"""GPU: the product-layer kernels exactly, at their chunk, tile and grid boundaries, with NaN in every padding.

The operands are small integers times a power of two, and every check first asserts, from the data, that the sum
of the absolute values of the terms of each result stays below 2^24 units of its grid.  Every partial sum in every
order is then exact in fp32, so the kernels must equal the float64 restatements (imported from the family tests)
bit for bit: a dropped, doubled or misplaced sample, k-slice, chunk or partial fails.

* b2ctr_bilinear (all three types), b2ctr_fefm, b2ctr_fwfm, b2ctr_pnn_inner (all four modes), b2ctr_pnn_outer,
  b2ctr_bi_interaction and b2ctr_regulate (copy / add / hadamard, with gates whose softmax is exact) at batch sizes
  taken from the library's own ``b2ctr_*_bwd_workspace_bytes``: B = 1, just below / at / just above the first
  chunk boundary, a B whose last chunks are empty, the C2 batch 65,536 and 65,537;
* x is the leading window of a wider buffer whose other columns, and the rows past the batch, hold NaN; outputs
  go into windows of NaN-filled buffers and incoming gradients are read from windows whose pitch gaps, other
  columns and extra rows hold NaN.  Results are finite, exact, and everything outside each window is unchanged
  bit for bit (NaN payloads included);
* E = 3 / 5 / 13 / 29 / 33 (one E that is not a multiple of 4 for each padded width EP): the NaN run equals the
  run with zero padding bit for bit;
* the clamped tile grid (65,535 tiles) goes round: bilinear, FEFM and PNN-outer forward and dx at F = 2 with
  B = 65535 * TS + r for E = 64 and E = 32, checked on the first and last two tiles and a strided sample of rows;
* the C2 production shapes of tools/pairwise_bench.py and tools/edcn_bench.py, exactly.
"""
import functools
import itertools

import pytest
import torch

import ccpm_oracle as CO
import flen_oracle as FO
import pnn_oracle as PO
from test_fefm_gpu import _ref_fefm, _ref_fwfm
from test_fibinet_gpu import _nw, _ref_bilinear
from test_pairwise_gpu import _ref_bi

pytestmark = pytest.mark.gpu

NAN_BITS = 0x7fc00123          # a quiet NaN with a payload, so a copy of it is told apart from a fresh NaN
EXTRA_ROWS = 3                 # rows past the batch in every buffer, all NaN
REF_ROWS = 8192                # float64 references in sample chunks of this many rows
TYPES = ("all", "each", "interaction")
PNN_MODES = ("inner", "elementwise", "vec", "num")


def _lib():
    from deepctr_b200 import _lib as L
    return L.lib()


# ------------------------------------------------------------------------------------------------ exact operands
def _grid(gen, shape, k, shift, device):
    """Integers in [-k, k] times 2^-shift (fp32)."""
    return torch.randint(-k, k + 1, tuple(shape), generator=gen, device=device, dtype=torch.float32).mul_(2.0 ** -shift)


def _nan_like(shape, device):
    return torch.full(tuple(shape), NAN_BITS, dtype=torch.int32, device=device).view(torch.float32)


def _padded(shape, device, fill):
    """A buffer of NaN (``fill`` None) or of ``fill``."""
    return _nan_like(shape, device) if fill is None else torch.full(tuple(shape), fill, device=device)


def _fits(bound, unit, what):
    """Every term a multiple of ``unit`` and sum |terms| < 2^24 units: every fp32 partial sum is exact."""
    top = float(bound.max()) if bound.numel() else 0.0
    assert top < 2.0 ** 24 * unit, "%s: the operands leave the exact range (%g >= 2^24 * %g)" % (what, top, unit)


def _same(got, want, what):
    """fp32 ``got`` equals the float64 ``want`` bit for bit (NaN never equals)."""
    g = got.double()
    bad = ~(g == want)
    n = int(bad.sum())
    if n:
        idx = tuple(int(i) for i in bad.nonzero()[0])
        raise AssertionError("%s: %d of %d entries differ, first at %s: got %r, want %r"
                             % (what, n, bad.numel(), idx, float(g[idx]), float(want[idx])))


class Window:
    """A [B, nblk, width] window at column ``col0`` of a [B + EXTRA_ROWS, ld] buffer of NaN (or ``fill``): block q
    at columns col0 + q * pitch.  ``check_outside`` asserts that nothing outside the window changed."""

    def __init__(self, B, ld, col0, nblk, width, pitch, device, fill=None):
        self.B, self.ld, self.col0, self.nblk, self.width, self.pitch = B, ld, col0, nblk, width, pitch
        assert col0 + (nblk - 1) * pitch + width <= ld
        self.fill_value = fill
        self.buf = _padded((B + EXTRA_ROWS, ld), device, fill)

    def blocks(self, t):
        base = t[:self.B, self.col0:]
        return torch.as_strided(base, (self.B, self.nblk, self.width), (t.stride(0), self.pitch, 1))

    def values(self):
        return self.blocks(self.buf)

    def fill(self, v):
        self.values()[...] = v
        return self

    def check_outside(self, what):
        """Put the padding value back into the window, compare the whole buffer with it, restore the window."""
        inside = self.values().clone()
        if self.fill_value is None:
            self.blocks(self.buf.view(torch.int32))[...] = NAN_BITS
            changed = self.buf.view(torch.int32) != NAN_BITS
        else:
            self.values()[...] = self.fill_value
            changed = self.buf != self.fill_value
        if bool(changed.any()):
            raise AssertionError("%s: %d entries outside the window were written" % (what, int(changed.count_nonzero())))
        del changed
        self.values()[...] = inside


def _digest(buf, rows=1024):
    """A fingerprint of a buffer's bits: per chunk of rows, the sum of its int32 bit patterns plain and weighted by
    position.  Cheap next to a copy of a multi-GB buffer, and any stray write of a different value changes it."""
    t = buf.view(torch.int32)
    out = []
    for r0 in range(0, t.shape[0], rows):
        c = t[r0:r0 + rows].to(torch.int64)
        w = torch.arange(1, c.numel() + 1, device=c.device).reshape(c.shape)
        out.append(torch.stack([c.sum(), (c * w).sum()]))
    return torch.stack(out)


class Frozen:
    """Buffers a kernel only reads: ``check`` asserts their bits are what they were when this was made."""

    def __init__(self, *bufs):
        self.bufs = bufs
        self.digests = [_digest(b) for b in bufs]

    def check(self, what):
        for k, (b, d) in enumerate(zip(self.bufs, self.digests)):
            assert torch.equal(_digest(b), d), "%s wrote into input buffer %d" % (what, k)


def _x_window(gen, B, F, E, device, k=2, shift=2, pad=11, fill=None):
    """x [B, F*E] on the grid as the leading window of a [B + EXTRA_ROWS, F*E + pad] buffer; the other columns and
    rows hold NaN (or ``fill``)."""
    ldx = F * E + pad
    buf = _padded((B + EXTRA_ROWS, ldx), device, fill)
    buf[:B, :F * E] = _grid(gen, (B, F * E), k, shift, device)
    return buf, buf[:B, :F * E], ldx


def _ref_pass(fn, x, g, weights, F, E, rows, absolute, visit):
    """float64 y = fn(x [b, F, E], *weights) and dx against the incoming gradient g (y's shape), handed to
    visit(rows slice, y [b, -1], dx [b, F*E]) in sample chunks; returns the weight gradients, accumulated over the
    chunks.  ``absolute``: on |x|, |g|, |weights|, which bounds every partial sum of a product of them."""
    B = x.shape[0]
    w64 = []
    for w in weights:
        w = w.double()
        w64.append((w.abs() if absolute else w).requires_grad_(True))
    for b0 in range(0, B, rows):
        sl = slice(b0, min(B, b0 + rows))
        x64, g64 = x[sl].double(), g[sl].double()
        if absolute:
            x64, g64 = x64.abs(), g64.abs()
        x64 = x64.reshape(-1, F, E).requires_grad_(True)
        y = fn(x64, *w64)
        (y * g64.reshape(y.shape)).sum().backward()
        visit(sl, y.detach().reshape(y.shape[0], -1), x64.grad.reshape(y.shape[0], -1))
    return [w.grad for w in w64]


def _exact_check(fn, x, g, weights, got, units, F, E, what, rows=REF_ROWS, bound_fn=None, check_dw=True):
    """Check that every result is in the exact range (units = (out, dx, dW) grid units), then that ``got`` = (y,
    dx, [dW per weight]) equals the float64 reference bit for bit.  The range comes from ``bound_fn`` (default
    ``fn``) on the absolute values, with its gradients: a sum of products with non-negative coefficients that
    dominates every partial sum the kernel forms.  ``check_dw`` False: out and dx only (weight gradients summed over
    more terms than the exact range holds)."""
    uy, udx, uw = units

    def bound(sl, y, dx):
        _fits(y, uy, what + " out")
        _fits(dx, udx, what + " dx")
    for k, w in enumerate(_ref_pass(bound_fn or fn, x, g, weights, F, E, rows, True, bound)):
        if check_dw:
            _fits(w, uw, "%s dW%d" % (what, k))
    gy, gdx, gdw = got

    def compare(sl, y, dx):
        if gy is not None:
            _same(gy[sl].reshape(y.shape), y, what + " out")
        _same(gdx[sl].reshape(dx.shape), dx, what + " dx")
    for k, (w, gw) in enumerate(zip(_ref_pass(fn, x, g, weights, F, E, rows, False, compare),
                                    gdw if check_dw else [])):
        _same(gw, w, "%s dW%d" % (what, k))


# ------------------------------------------------------------------------------------------------ chunk boundaries
def _per(B, nchunk):
    return -(-B // nchunk)


def _chunk_batches(nchunk, step):
    """Batch sizes for a reduction split into nchunk(B) chunks of at least ``step`` samples: 1, step - 1, step,
    step + 1 (asserting that the chunk count moves there), the first B whose last chunk is empty, 65536 and 65537."""
    assert nchunk(1) == nchunk(step - 1) == nchunk(step) == 1 and nchunk(step + 1) == 2, \
        "the first chunk boundary is not at %d samples" % step
    empty = next((B for B in range(step + 2, 1 << 18)
                  if nchunk(B) > 1 and _per(B, nchunk(B)) * (nchunk(B) - 1) >= B), None)
    assert empty is not None, "no batch below 2^18 leaves the last chunk empty"
    return [1, step - 1, step, step + 1, empty, 65536, 65537]


@functools.lru_cache(maxsize=None)
def _batches_for(kind, F, E, mode=None):
    """A family's batch list, derived from its b2ctr_*_bwd_workspace_bytes (host functions: no device needed)."""
    L = _lib()
    P = F * (F - 1) // 2
    if kind == "bi":           # bilinear, FEFM and PNN 'mat': [nchunk][P][E][E] partials, >= kBiDwSub = 64 a chunk
        return _chunk_batches(lambda B: L.b2ctr_bilinear_bwd_workspace_bytes(F, E, B) // (P * E * E * 4), 64)
    if kind == "pnn":          # PNN vec / num: [nchunk][entries] partials, >= 64 samples a chunk
        from deepctr_b200 import kernels as K
        nent = P * E if mode == "vec" else P
        return _chunk_batches(
            lambda B: L.b2ctr_pnn_inner_bwd_workspace_bytes(F, E, K.PNN_MODES[mode], B) // (nent * 4), 64)
    if kind == "reg":          # regulate: [nchunk + 1][2][F], >= 128 samples a chunk
        return _chunk_batches(lambda B: L.b2ctr_regulate_bwd_workspace_bytes(F, E, B) // (2 * F * 4) - 1, 128)
    raise KeyError(kind)


CHUNK_CASES = ["one", "below", "at", "above", "empty_last", "c2", "c2_plus_1"]


# ------------------------------------------------------------------------------------------------ bilinear
def _bilinear_case(cuda, B, F, E, t, seed, pitch=None, col0=3, fill=None):
    """Forward into pair windows of pitch ``pitch`` of a NaN buffer, backward from a NaN-padded gradient window."""
    from deepctr_b200 import kernels as K
    gen = torch.Generator(device=cuda).manual_seed(seed)
    P = F * (F - 1) // 2
    pitch = pitch or E + 3
    xbuf, xw, ldx = _x_window(gen, B, F, E, cuda, fill=fill)
    W = _grid(gen, (_nw(t, F), E, E), 3, 1, cuda)
    ld = col0 + (P - 1) * pitch + E + 2
    out = Window(B, ld, col0, P, E, pitch, cuda, fill)
    K.bilinear_fwd(xw, ldx, F, E, t, W, B, out=out.buf, col0=col0, pitch=pitch)
    out.check_outside("bilinear_fwd")
    gwin = Window(B, ld, col0, P, E, pitch, cuda, fill).fill(_grid(gen, (B, P, E), 3, 2, cuda))
    frozen = Frozen(xbuf, gwin.buf)
    dx, dW = K.bilinear_bwd(gwin.buf, ld, col0, pitch, xw, ldx, F, E, t, W, B)
    frozen.check("bilinear_bwd")
    return dict(x=xw, W=W, out=out.values(), g=gwin.values(), dx=dx, dW=dW)


def _check_bilinear_exact(r, F, E, t):
    # out: x (1/4) * W (1/2) * x (1/4) -> 1/32;  dx: g (1/4) * W * x -> 1/32;  dW: x * g * x -> 1/64
    _exact_check(lambda x, W: _ref_bilinear(x, t, W), r["x"], r["g"], [r["W"]], (r["out"], r["dx"], [r["dW"]]),
                 (2.0 ** -5, 2.0 ** -5, 2.0 ** -6), F, E, "bilinear " + t)


BI_FE = [(3, 5), (3, 32)]


@pytest.mark.parametrize("case", range(len(CHUNK_CASES)), ids=CHUNK_CASES)
@pytest.mark.parametrize("t", TYPES)
@pytest.mark.parametrize("F,E", BI_FE)
def test_bilinear_exact_at_chunk_boundaries(cuda, F, E, t, case):
    B = _batches_for("bi", F, E)[case]
    _check_bilinear_exact(_bilinear_case(cuda, B, F, E, t, seed=B + E), F, E, t)


# ------------------------------------------------------------------------------------------------ FEFM / PNN outer
def _ref_mat(x, Kw):
    return PO.outer(x, Kw, "mat")


def _fefm_case(cuda, B, F, E, seed, col0=5, kind="fefm", fill=None, ld=None, ldx_pad=11):
    """FEFM (S = W + W^T through fefm_sym) or PNN 'mat' (K [E, P, E]): scores into a column window of a NaN
    buffer, the gradient read from a window of another."""
    from deepctr_b200 import kernels as K
    gen = torch.Generator(device=cuda).manual_seed(seed)
    P = F * (F - 1) // 2
    xbuf, xw, ldx = _x_window(gen, B, F, E, cuda, fill=fill, pad=ldx_pad)
    if kind == "fefm":
        W = _grid(gen, (P, E, E), 3, 2, cuda)
        M = K.fefm_sym(W)
        fwd, bwd = K.fefm_fwd, K.fefm_bwd
    else:
        W = M = _grid(gen, (E, P, E), 3, 1, cuda)
        fwd, bwd = K.pnn_outer_fwd, K.pnn_outer_bwd
    ld = ld or col0 + P + 4
    out = Window(B, ld, col0, 1, P, P, cuda, fill)
    fwd(xw, ldx, F, E, M, B, out=out.buf, col0=col0)
    out.check_outside(kind + " fwd")
    gwin = Window(B, ld, col0, 1, P, P, cuda, fill).fill(_grid(gen, (B, 1, P), 3, 2, cuda))
    frozen = Frozen(xbuf, gwin.buf)
    dx, dW = bwd(gwin.buf, ld, col0, xw, ldx, F, E, M, B)
    frozen.check(kind + " bwd")
    return dict(x=xw, W=W, out=out.values(), g=gwin.values(), dx=dx, dW=dW)


def _check_fefm_exact(r, F, E, kind):
    # fefm: x (1/4) S (1/4) x -> 1/64 for out, dx and dW;  mat: K in 1/2 -> out, dx 1/32, dK 1/64
    fn = _ref_fefm if kind == "fefm" else _ref_mat
    u = 2.0 ** -6 if kind == "fefm" else 2.0 ** -5
    _exact_check(fn, r["x"], r["g"], [r["W"]], (r["out"], r["dx"], [r["dW"]]), (u, u, 2.0 ** -6), F, E, kind)


@pytest.mark.parametrize("case", range(len(CHUNK_CASES)), ids=CHUNK_CASES)
@pytest.mark.parametrize("kind", ["fefm", "mat"])
@pytest.mark.parametrize("F,E", BI_FE)
def test_fefm_and_pnn_outer_exact_at_chunk_boundaries(cuda, F, E, kind, case):
    B = _batches_for("bi", F, E)[case]        # both use the bilinear weight-gradient chunks
    L = _lib()
    assert (L.b2ctr_fefm_bwd_workspace_bytes(F, E, B) == L.b2ctr_pnn_outer_bwd_workspace_bytes(F, E, B)
            == L.b2ctr_bilinear_bwd_workspace_bytes(F, E, B))
    _check_fefm_exact(_fefm_case(cuda, B, F, E, seed=3 * B + E, kind=kind), F, E, kind)


# ------------------------------------------------------------------------------------------------ PNN inner
def _pnn_case(cuda, B, F, E, mode, seed, col0=2, fill=None, ld=None, ldx_pad=11):
    from deepctr_b200 import kernels as K
    gen = torch.Generator(device=cuda).manual_seed(seed)
    P = F * (F - 1) // 2
    xbuf, xw, ldx = _x_window(gen, B, F, E, cuda, fill=fill, pad=ldx_pad)
    Kw = _grid(gen, (P, E) if mode == "vec" else (P, 1), 3, 1, cuda) if mode in ("vec", "num") else None
    width = P * E if mode == "elementwise" else P
    ld = ld or col0 + width + 3
    out = Window(B, ld, col0, 1, width, width, cuda, fill)
    K.pnn_inner_fwd(xw, ldx, F, E, mode, Kw, B, out=out.buf, col0=col0)
    out.check_outside("pnn_inner_fwd " + mode)
    gwin = Window(B, ld, col0, 1, width, width, cuda, fill).fill(_grid(gen, (B, 1, width), 3, 2, cuda))
    frozen = Frozen(xbuf, gwin.buf)
    dx, dK = K.pnn_inner_bwd(gwin.buf, ld, col0, xw, ldx, F, E, mode, Kw, B)
    frozen.check("pnn_inner_bwd " + mode)
    return dict(x=xw, W=Kw, out=out.values(), g=gwin.values(), dx=dx, dW=dK)


def _check_pnn_exact(r, F, E, mode):
    # x (1/4) x (1/4) [K (1/2)] -> 1/32 at most; dx g (1/4) [K] x -> 1/32; dK g x x -> 1/64
    if mode in ("inner", "elementwise"):
        assert r["dW"] is None
        fn, weights, dws = (lambda x: PO.inner(x, mode == "inner").flatten(1)), [], []
    else:
        fn, weights, dws = (lambda x, Kw: PO.outer(x, Kw, mode)), [r["W"]], [r["dW"]]
    _exact_check(fn, r["x"], r["g"], weights, (r["out"], r["dx"], dws), (2.0 ** -5, 2.0 ** -5, 2.0 ** -6), F, E,
                 "pnn " + mode)


@pytest.mark.parametrize("case", range(len(CHUNK_CASES)), ids=CHUNK_CASES)
@pytest.mark.parametrize("mode", PNN_MODES)
@pytest.mark.parametrize("F,E", [(3, 5), (9, 32)])
def test_pnn_inner_exact_at_chunk_boundaries(cuda, F, E, mode, case):
    # inner / elementwise have no kernel gradient: they run at the batches of 'vec'
    B = _batches_for("pnn", F, E, mode if mode in ("vec", "num") else "vec")[case]
    _check_pnn_exact(_pnn_case(cuda, B, F, E, mode, seed=5 * B + E), F, E, mode)


# ------------------------------------------------------------------------------------------------ FwFM
# dR partials are per CTA: kFwWarps = 8 samples a round, grid_for(B, 8, 4) = min(ceil(B / 8), 528) CTAs
FWFM_BATCHES = [1, 7, 8, 9, 528 * 8 - 1, 528 * 8, 528 * 8 + 1, 65536, 65537]


def _fwfm_case(cuda, B, F, E, seed, fill=None, ldx_pad=11):
    from deepctr_b200 import kernels as K
    gen = torch.Generator(device=cuda).manual_seed(seed)
    xbuf, xw, ldx = _x_window(gen, B, F, E, cuda, fill=fill, pad=ldx_pad)
    r = _grid(gen, (F, F), 3, 1, cuda)
    out = K.fwfm_fwd(xw, ldx, F, E, r, B)
    gwin = Window(B, 3, 1, 1, 1, 1, cuda, fill).fill(_grid(gen, (B, 1, 1), 3, 2, cuda))
    frozen = Frozen(xbuf, gwin.buf)
    dx, dR = K.fwfm_bwd(gwin.buf[:, 1:2], 3, xw, ldx, F, E, r, B)
    frozen.check("fwfm_bwd")
    return dict(x=xw, W=r, out=out, g=gwin.values(), dx=dx, dW=dR)


def _check_fwfm_exact(r, F, E):
    _exact_check(_ref_fwfm, r["x"], r["g"], [r["W"]], (r["out"], r["dx"], [r["dW"]]),
                 (2.0 ** -5, 2.0 ** -5, 2.0 ** -6), F, E, "fwfm")


@pytest.mark.parametrize("B", FWFM_BATCHES, ids=["B%d" % b for b in FWFM_BATCHES])
@pytest.mark.parametrize("F,E", [(3, 5), (26, 32)])
def test_fwfm_exact_at_block_boundaries(cuda, F, E, B):
    """B around one CTA's round of 8 samples and around the grid cap, where the grid-stride loop starts to go
    round; the CTA count is the workspace's partial count."""
    P = F * (F - 1) // 2
    nb = lambda b: _lib().b2ctr_fwfm_bwd_workspace_bytes(F, b) // (P * 4)      # noqa: E731
    assert nb(8) == 1 and nb(9) == 2 and nb(528 * 8 - 1) == nb(528 * 8) == nb(528 * 8 + 1) == nb(65537) == 528
    _check_fwfm_exact(_fwfm_case(cuda, B, F, E, seed=7 * B + F), F, E)


# ------------------------------------------------------------------------------------------------ Bi-Interaction
def _bi_case(cuda, B, F, E, seed, fill=None):
    from deepctr_b200 import kernels as K
    gen = torch.Generator(device=cuda).manual_seed(seed)
    xbuf, xw, ldx = _x_window(gen, B, F, E, cuda, fill=fill)
    gwin = Window(B, E + 6, 2, 1, E, E, cuda, fill).fill(_grid(gen, (B, 1, E), 3, 2, cuda))
    out = K.bi_interaction_fwd(xw, ldx, F, E, B)
    frozen = Frozen(xbuf, gwin.buf)
    dx = K.bi_interaction_bwd(xw, ldx, F, E, gwin.buf[:B, 2:2 + E], B)
    frozen.check("bi_interaction_bwd")
    return dict(x=xw, out=out, g=gwin.values(), dx=dx)


def _check_bi_exact(r, F, E):
    # the kernel forms s = sum_f x and q = sum_f x^2 (1/16): (sum |x|)^2 + sum x^2 and |g| (sum |x| + |x|) bound
    # every partial
    ax = r["x"].double().abs().reshape(-1, F, E)
    _fits(ax.sum(1) ** 2 + (ax * ax).sum(1), 2.0 ** -4, "bi_interaction out")
    _fits(r["g"].double().abs().reshape(-1, 1, E) * (ax.sum(1, keepdim=True) + ax), 2.0 ** -4, "bi_interaction dx")

    def compare(sl, y, dx):
        _same(r["out"][sl], y, "bi_interaction_fwd")
        _same(r["dx"][sl], dx, "bi_interaction_bwd")
    _ref_pass(_ref_bi, r["x"], r["g"], [], F, E, REF_ROWS, False, compare)


BI_BATCHES = [1, 255, 256, 257, 65537]


@pytest.mark.parametrize("B", BI_BATCHES, ids=["B%d" % b for b in BI_BATCHES])
@pytest.mark.parametrize("F,E", [(2, 4), (26, 32), (7, 33)])
def test_bi_interaction_exact(cuda, F, E, B):
    _check_bi_exact(_bi_case(cuda, B, F, E, seed=B + F * E), F, E)


# ------------------------------------------------------------------------------------------------ EDCN regulate
def _exact_gates(F, seed, cuda, on=None):
    """Gate weights whose softmax is exact: ``on`` fields (a power of two, default the largest one <= F, so every
    field when F is a power of two) at 0, the others at -1e4, where expf underflows to 0: the gates are 1/on or 0.
    -> (weights [F], float64 gates [F])."""
    on = on or 1 << (F.bit_length() - 1)
    idx = torch.randperm(F, generator=torch.Generator().manual_seed(seed))[:on].to(cuda)
    g = torch.full((F,), -1e4, device=cuda)
    g[idx] = 0.0
    gates = torch.zeros(F, dtype=torch.float64, device=cuda)
    gates[idx] = 1.0 / on
    return g, gates


REG_MODES = ("copy", "add", "hadamard", "attention")


def _regulate_case(cuda, B, F, E, mode, seed, accumulate, fill=None, on=None):
    """u, y0 and y1 into windows of NaN buffers; backward from NaN-padded du / dy0 / dy1 windows into a dx window
    of a NaN buffer (accumulating: the window holds grid values), with dh (dax, dah) and both gate gradients.  The
    incoming gradients are in [-1/4, 1/4], which keeps the gate-gradient sums of 135,169 samples exact."""
    from deepctr_b200 import kernels as K
    gen = torch.Generator(device=cuda).manual_seed(seed)
    d = F * E
    # x, h, and the attention weights ax, ah (in [-1/4, 1/4]), each a window of its own NaN-padded buffer
    n_in = 4 if mode == "attention" else 1 if mode == "copy" else 2
    ins = [_x_window(gen, B, F, E, cuda, k=2 if i < 2 else 1, pad=8 + 4 * i, fill=fill) for i in range(n_in)]
    xw, hw, axw, ahw = ([w for _, w, _ in ins] + [None] * 3)[:4]
    (g0, gate0), (g1, gate1) = _exact_gates(F, seed, cuda, on), _exact_gates(F, seed + 1, cuda, on)
    gates = [(g0, 1.0), (g1, 1.0)]
    outs = [Window(B, d + 12, c, 1, d, d, cuda, fill) for c in (4, 8, 0)]
    K.regulate_fwd(mode, F, E, B, xw, hw, axw, ahw, gates, u=(outs[0].buf, 4), y0=(outs[1].buf, 8),
                   y1=(outs[2].buf, 0))
    for o, n in zip(outs, ("u", "y0", "y1")):
        o.check_outside("regulate_fwd " + n)
    grads = [Window(B, d + 8, c, 1, d, d, cuda, fill).fill(_grid(gen, (B, 1, d), 1, 2, cuda)) for c in (4, 0, 8)]
    dxw = Window(B, d + 8, 4, 1, d, d, cuda, fill)
    if accumulate:
        dxw.fill(_grid(gen, (B, 1, d), 3, 2, cuda))
    dx0 = dxw.values().clone()
    frozen = Frozen(*[buf for buf, _, _ in ins], *[gw.buf for gw in grads])
    _, dh, dax, dah, dg0, dg1 = K.regulate_bwd(
        mode, F, E, B, xw, hw, axw, ahw, gates, du=(grads[0].buf, 4), dy0=(grads[1].buf, 0),
        dy1=(grads[2].buf, 8), dx=dxw.buf[:B, 4:4 + d], dx_accumulate=accumulate, want_dh=mode != "copy",
        want_dax=mode == "attention", want_dah=mode == "attention", want_dg=(True, True))
    frozen.check("regulate_bwd " + mode)
    dxw.check_outside("regulate_bwd dx")
    return dict(x=xw, h=hw, ax=axw, ah=ahw, gates=(gate0, gate1), outs=[o.values().reshape(B, d) for o in outs],
                grads=[gw.values().reshape(B, d) for gw in grads], dx=dxw.values().reshape(B, d),
                dx0=dx0.reshape(B, d), dh=dh, dax=dax, dah=dah, dg=(dg0, dg1))


def _check_regulate_exact(r, F, E, mode, accumulate):
    B, d = r["x"].shape
    x, h, ax, ah = (r[k].double() if r[k] is not None else None for k in ("x", "h", "ax", "ah"))
    v = {"copy": lambda: x, "add": lambda: x + h, "hadamard": lambda: x * h,
         "attention": lambda: ax * x + ah * h}[mode]()
    du, dy0, dy1 = (t.double() for t in r["grads"])
    gate = [gk.repeat_interleave(E)[None, :] for gk in r["gates"]]
    _same(r["outs"][0], v, "regulate u")
    _same(r["outs"][1], v * gate[0], "regulate y0")
    _same(r["outs"][2], v * gate[1], "regulate y1")
    dv = du + gate[0] * dy0 + gate[1] * dy1
    dxw = dv * h if mode == "hadamard" else dv * ax if mode == "attention" else dv
    _same(r["dx"], dxw + (r["dx0"].double() if accumulate else 0), "regulate dx")
    if mode != "copy":
        _same(r["dh"], dv * x if mode == "hadamard" else dv * ah if mode == "attention" else dv, "regulate dh")
    if mode == "attention":
        _same(r["dax"], dv * x, "regulate dax")
        _same(r["dah"], dv * h, "regulate dah")
    # dg_k = gate_k * (s_k - <gate_k, s_k>), s_k[f] = sum_b sum_e v dy_k (1/16 for copy and add, else 1/64): exact
    # with these gates while the sum over the gated fields of sum |v dy_k| stays in range
    unit = 2.0 ** -4 if mode in ("copy", "add") else 2.0 ** -6
    vabs = x.abs() if mode == "copy" else x.abs() + h.abs() if mode == "add" else \
        (x * h).abs() if mode == "hadamard" else (ax * x).abs() + (ah * h).abs()
    for k, (dy, gk, dg) in enumerate(zip((dy0, dy1), r["gates"], r["dg"])):
        sabs = (vabs * dy.abs()).reshape(B, F, E).sum(dim=(0, 2))
        _fits(2 * (sabs * (gk > 0)).sum(), unit, "regulate s%d" % k)
        s = (v * dy).reshape(B, F, E).sum(dim=(0, 2))
        _same(dg, gk * (s - (gk * s).sum()), "regulate dg%d" % k)


@pytest.mark.parametrize("case", range(len(CHUNK_CASES)), ids=CHUNK_CASES)
@pytest.mark.parametrize("mode", REG_MODES)
@pytest.mark.parametrize("F,E", [(8, 4), (6, 5)])
def test_regulate_exact_at_chunk_boundaries(cuda, F, E, mode, case):
    """E = 4: the float4 path, E = 5: the scalar path; dx written on odd cases, added to on even ones."""
    B = _batches_for("reg", F, E)[case]
    acc = case % 2 == 0
    _check_regulate_exact(_regulate_case(cuda, B, F, E, mode, seed=B + F, accumulate=acc), F, E, mode, acc)


# ------------------------------------------------------------------------------------------------ NaN padding
PAD_E = [3, 5, 13, 29, 33]          # EP = 4 / 8 / 16 / 32 / 64, none a multiple of 4


def _nan_equals_zero_padding(make, keys):
    """make(fill) runs a case with ``fill`` (None: NaN) in every padding; the results are finite and the runs agree
    bit for bit."""
    def flat(r):
        out = []
        for k in keys:
            t = r[k]
            out += list(t) if isinstance(t, (list, tuple)) else [t]
        return [t for t in out if t is not None]
    a, b = flat(make(None)), flat(make(0.0))
    assert len(a) == len(b) and a
    for u, w in zip(a, b):
        assert bool(torch.isfinite(u).all()), "a NaN in the padding reached a result"
        assert torch.equal(u.contiguous().view(torch.int32), w.contiguous().view(torch.int32))


@pytest.mark.parametrize("E", PAD_E)
@pytest.mark.parametrize("t", TYPES)
def test_bilinear_nan_padding(cuda, t, E):
    F, B = 4, 133
    _check_bilinear_exact(_bilinear_case(cuda, B, F, E, t, seed=E), F, E, t)
    _nan_equals_zero_padding(lambda fill: _bilinear_case(cuda, B, F, E, t, seed=E, fill=fill), ("out", "dx", "dW"))


@pytest.mark.parametrize("E", PAD_E)
@pytest.mark.parametrize("kind", ["fefm", "mat"])
def test_fefm_and_pnn_outer_nan_padding(cuda, kind, E):
    F, B = 5, 133
    _check_fefm_exact(_fefm_case(cuda, B, F, E, seed=E, kind=kind), F, E, kind)
    _nan_equals_zero_padding(lambda fill: _fefm_case(cuda, B, F, E, seed=E, kind=kind, fill=fill), ("out", "dx", "dW"))


@pytest.mark.parametrize("E", PAD_E)
@pytest.mark.parametrize("mode", PNN_MODES)
def test_pnn_inner_nan_padding(cuda, mode, E):
    F, B = 5, 133
    _check_pnn_exact(_pnn_case(cuda, B, F, E, mode, seed=E), F, E, mode)
    _nan_equals_zero_padding(lambda fill: _pnn_case(cuda, B, F, E, mode, seed=E, fill=fill), ("out", "dx", "dW"))


@pytest.mark.parametrize("E", PAD_E)
def test_fwfm_and_bi_interaction_nan_padding(cuda, E):
    F, B = 5, 133
    _check_fwfm_exact(_fwfm_case(cuda, B, F, E, seed=E), F, E)
    _nan_equals_zero_padding(lambda fill: _fwfm_case(cuda, B, F, E, seed=E, fill=fill), ("out", "dx", "dW"))
    _check_bi_exact(_bi_case(cuda, B, F, E, seed=E), F, E)
    _nan_equals_zero_padding(lambda fill: _bi_case(cuda, B, F, E, seed=E, fill=fill), ("out", "dx"))


@pytest.mark.parametrize("E", PAD_E + [4, 16])
@pytest.mark.parametrize("mode", REG_MODES)
def test_regulate_nan_padding(cuda, mode, E):
    F, B = 4, 133
    for acc in (False, True):
        _check_regulate_exact(_regulate_case(cuda, B, F, E, mode, seed=E, accumulate=acc), F, E, mode, acc)
    _nan_equals_zero_padding(lambda fill: _regulate_case(cuda, B, F, E, mode, seed=E, accumulate=True, fill=fill),
                             ("outs", "dx", "dh", "dax", "dah", "dg"))


# ------------------------------------------------------------------------------------------------ clamped grid
def _clamp_rows(B, TS, device):
    """The first and last two tiles in full and every 4099th row."""
    nt = -(-B // TS)
    rows = torch.cat([torch.arange(0, 2 * TS), torch.arange((nt - 2) * TS, B), torch.arange(2 * TS, B, 4099)])
    return torch.unique(rows).to(device)


@pytest.mark.parametrize("E,B", [(64, 65535 * 64 + 37), (32, 65535 * 128 + 5)], ids=["E64", "E32"])
def test_clamped_tile_grid_goes_round(cuda, E, B):
    """F = 2: one pair, tiles of TS = 4096 / E samples, 65,536 tiles on a grid clamped to 65,535, so the CTAs of
    tile 0 also take the last, partial tile.  Bilinear (three types), FEFM and PNN-outer forward and dx."""
    from deepctr_b200 import kernels as K
    F, TS = 2, 4096 // E
    assert -(-B // TS) == 65536 and B % TS
    gen = torch.Generator(device=cuda).manual_seed(E)
    x = _grid(gen, (B, F * E), 2, 2, cuda)
    rows = _clamp_rows(B, TS, cuda)
    xs = x[rows]
    units = (2.0 ** -5, 2.0 ** -5, 2.0 ** -6)
    for t in TYPES:
        W = _grid(gen, (1, E, E), 3, 1, cuda)
        out = K.bilinear_fwd(x, F * E, F, E, t, W, B)
        g = _grid(gen, (B, E), 3, 2, cuda)
        dx, _ = K.bilinear_bwd(g, E, 0, E, x, F * E, F, E, t, W, B, want_dw=False)
        _exact_check(lambda x_, W_: _ref_bilinear(x_, t, W_), xs, g[rows], [W], (out[rows], dx[rows], []), units,
                     F, E, "bilinear %s (clamped grid)" % t)
        del out, g, dx
    for kind in ("fefm", "mat"):
        if kind == "fefm":
            W = _grid(gen, (1, E, E), 3, 2, cuda)
            M = K.fefm_sym(W)
            out = K.fefm_fwd(x, F * E, F, E, M, B)
            g = _grid(gen, (B, 1), 3, 2, cuda)
            dx, _ = K.fefm_bwd(g, 1, 0, x, F * E, F, E, M, B, want_dw=False)
            fn, u = _ref_fefm, (2.0 ** -6,) * 3
        else:
            W = _grid(gen, (E, 1, E), 3, 1, cuda)
            out = K.pnn_outer_fwd(x, F * E, F, E, W, B)
            g = _grid(gen, (B, 1), 3, 2, cuda)
            dx, _ = K.pnn_outer_bwd(g, 1, 0, x, F * E, F, E, W, B, want_dk=False)
            fn, u = _ref_mat, units
        _exact_check(fn, xs, g[rows], [W], (out[rows], dx[rows], []), u, F, E, "%s (clamped grid)" % kind)
        del out, g, dx


# ------------------------------------------------------------------------------------------------ production shapes
def test_c2_bilinear_placed_in_the_dnn_input(cuda):
    """tools/pairwise_bench.py's FiBiNET case: B = 65536, F = 26, E = 32, x a window of a [B, 848] buffer, the
    'interaction' pairs at pitch 2E in the [B, 20816] DNN input, and the gradient read from the other half of every
    pair slot, as the bench does."""
    from deepctr_b200 import kernels as K
    B, F, E = 65536, 26, 32
    P = F * (F - 1) // 2
    ld = (2 * P * E + 13 + 3) // 4 * 4
    gen = torch.Generator(device=cuda).manual_seed(11)
    xbuf, xw, ldx = _x_window(gen, B, F, E, cuda, pad=848 - F * E)
    W = _grid(gen, (P, E, E), 3, 1, cuda)
    dnn = Window(B, ld, 0, P, E, 2 * E, cuda)
    K.bilinear_fwd(xw, ldx, F, E, "interaction", W, B, out=dnn.buf, col0=0, pitch=2 * E)
    dnn.check_outside("bilinear_fwd (C2)")
    out = dnn.values().clone()
    g = torch.as_strided(dnn.buf[:B, E:], (B, P, E), (ld, 2 * E, 1))
    for b0 in range(0, B, REF_ROWS):
        g[b0:b0 + REF_ROWS] = _grid(gen, (min(B - b0, REF_ROWS), P, E), 3, 2, cuda)
    frozen = Frozen(xbuf, dnn.buf)
    dx, dW = K.bilinear_bwd(dnn.buf, ld, E, 2 * E, xw, ldx, F, E, "interaction", W, B)
    frozen.check("bilinear_bwd (C2)")
    _exact_check(lambda x_, W_: _ref_bilinear(x_, "interaction", W_), xw, g, [W], (out, dx, [dW]),
                 (2.0 ** -5, 2.0 ** -5, 2.0 ** -6), F, E, "bilinear (C2)", rows=2048)


@pytest.mark.parametrize("kind", ["fefm", "mat", "inner", "vec", "num", "fwfm"])
def test_c2_scores_placed_in_the_dnn_input(cuda, kind):
    """tools/pairwise_bench.py's DeepFEFM / PNN / FwFM cases: B = 65536, F = 26, E = 32, x a window of the [B, 848]
    gather buffer, the 325 scores at column 845 of a [B, 1172] buffer and their gradient read from there."""
    B, F, E, pad = 65536, 26, 32, 848 - 832
    if kind in ("fefm", "mat"):
        _check_fefm_exact(_fefm_case(cuda, B, F, E, seed=12, col0=845, kind=kind, ld=1172, ldx_pad=pad), F, E, kind)
    elif kind == "fwfm":
        _check_fwfm_exact(_fwfm_case(cuda, B, F, E, seed=12, ldx_pad=pad), F, E)
    else:
        _check_pnn_exact(_pnn_case(cuda, B, F, E, kind, seed=12, col0=845, ld=1172, ldx_pad=pad), F, E, kind)


@pytest.mark.parametrize("mode", REG_MODES)
def test_edcn_bench_shape_regulate(cuda, mode):
    """tools/edcn_bench.py: B = 65536, 26 fields, E = 16, dx added into an existing gradient.  Two fields per gate
    are on (softmax 1/2 exactly): the gate-gradient sums of 65,536 x 16 terms per field stay exact for two."""
    _check_regulate_exact(_regulate_case(cuda, 65536, 26, 16, mode, seed=13, accumulate=True, on=2), 26, 16, mode,
                          True)


def test_bi_interaction_c2_shape(cuda):
    """tools/pairwise_bench.py's NFM case: B = 65536, F = 26, E = 32."""
    _check_bi_exact(_bi_case(cuda, 65536, 26, 32, seed=14), 26, 32)


# ------------------------------------------------------------------------------------------------ FLEN
def _fwbi_nchunk(cuda, sizes, E):
    """nchunk(B) of b2ctr_field_wise_bi_bwd, from its workspace function: [nchunk][P + G + E] partials."""
    import ctypes
    from deepctr_b200 import kernels as K
    G = len(sizes)
    F, P = sum(sizes), G * (G - 1) // 2
    t = torch.zeros((1, F * E + E), device=cuda)
    k = torch.zeros((max(P, 1), 1), device=cuda)
    a = K._fwbi_desc(t, [f * E for f in range(F)], [f % G for f in range(F)], G, E, 1, k, k, None, None, t, 0)
    a.dkernel_mf = k.data_ptr()

    def nchunk(B):
        a.batch = B
        return _lib().b2ctr_field_wise_bi_bwd_workspace_bytes(ctypes.byref(a)) // ((P + G + E) * 4)
    return nchunk


def _fwbi_case(cuda, B, sizes, E, seed, use_bias=True, accumulate=False, fill=None, offset=3):
    """FieldWiseBiInteraction on fields at column ``offset`` of a NaN-padded buffer (group of field f: interleaved
    over the groups), h into a column window of a NaN buffer, dh read from a NaN-padded window, dx written (or
    added) into the fields' columns of a NaN buffer.  x and dh in [-1/4, 1/4], the kernels in 1/2 steps."""
    from deepctr_b200 import kernels as K
    gen = torch.Generator(device=cuda).manual_seed(seed)
    G = len(sizes)
    order = [g for r in range(max(sizes)) for g in range(G) if r < sizes[g]]
    F, P = len(order), G * (G - 1) // 2
    cols = [offset + f * E for f in range(F)]
    ldx = offset + F * E + 5
    xbuf = _padded((B + EXTRA_ROWS, ldx), cuda, fill)
    xbuf[:B, offset:offset + F * E] = _grid(gen, (B, F * E), 1, 2, cuda)
    kmf, kfm = _grid(gen, (P, 1), 3, 1, cuda), _grid(gen, (G, 1), 3, 1, cuda)
    bmf, bfm = (_grid(gen, (E,), 3, 2, cuda), _grid(gen, (E,), 3, 2, cuda)) if use_bias else (None, None)
    out = Window(B, E + 4, 2, 1, E, E, cuda, fill)
    K.field_wise_bi_fwd(xbuf, cols, order, G, E, B, kmf, kfm, bmf, bfm, out.buf, outcol=2)
    out.check_outside("field_wise_bi_fwd")
    dh = Window(B, E + 3, 1, 1, E, E, cuda, fill).fill(_grid(gen, (B, 1, E), 1, 2, cuda))
    dxw = Window(B, ldx, offset, 1, F * E, F * E, cuda, fill)
    if accumulate:
        dxw.fill(_grid(gen, (B, 1, F * E), 3, 2, cuda))
    dx0 = dxw.values().clone()
    frozen = Frozen(xbuf, dh.buf)
    dws = K.field_wise_bi_bwd(xbuf, cols, order, G, E, B, kmf, kfm, bmf, bfm, dh.buf, doutcol=1, dx=dxw.buf,
                              dx_accumulate=accumulate, want_dkernel=(True, True), want_dbias=(use_bias, use_bias))
    frozen.check("field_wise_bi_bwd")
    dxw.check_outside("field_wise_bi_bwd dx")
    weights = [kmf, kfm] + ([bmf, bfm] if use_bias else [])
    return dict(x=xbuf[:B, offset:offset + F * E], order=order, G=G, weights=weights, out=out.values(),
                g=dh.values(), dx=dxw.values(), dx0=dx0, dW=[w for w in dws if w is not None])


def _check_fwbi_exact(r, E, accumulate, check_dw=True):
    G, order = r["G"], r["order"]
    F = len(order)
    idx = [[f for f in range(F) if order[f] == g] for g in range(G)]

    def fn(x, *w):
        return FO.field_wise_bi([x[:, i] for i in idx], *w)

    def bound(x, kmf, kfm, *b):
        # |kmf| S_g S_h + |kfm| (S_g^2 + Q_g) + |biases| on |x|: bounds S, Q, S^2 - Q, every fma and their sums
        S = [x[:, i].sum(1) for i in idx]
        Q = [(x[:, i] * x[:, i]).sum(1) for i in idx]
        y = sum(kmf[p, 0] * S[i] * S[j] for p, (i, j) in enumerate(itertools.combinations(range(G), 2)))
        y = y + sum(kfm[g, 0] * (S[g] * S[g] + Q[g]) for g in range(G))
        return y + sum(b) if b else y
    dx = r["dx"].reshape(r["dx"].shape[0], -1)
    if accumulate:
        dx = dx - r["dx0"].reshape(dx.shape)          # exact: both terms and the sum are on the grid
    _exact_check(fn, r["x"], r["g"], r["weights"], (r["out"], dx, r["dW"]),
                 (2.0 ** -5, 2.0 ** -5, 2.0 ** -6), F, E, "field_wise_bi", bound_fn=bound, check_dw=check_dw)


@pytest.mark.parametrize("case", range(len(CHUNK_CASES)), ids=CHUNK_CASES)
@pytest.mark.parametrize("use_bias", [False, True], ids=["nobias", "bias"])
@pytest.mark.parametrize("sizes,E", [((2, 1, 1), 4), ((1, 2), 3)], ids=["G3_E4", "G2_E3"])
def test_field_wise_bi_exact_at_chunk_boundaries(cuda, sizes, E, use_bias, case):
    """E = 4: the float4 path, E = 3: the scalar one; dx added on even cases, written on odd ones."""
    B = _chunk_batches(_fwbi_nchunk(cuda, sizes, E), 128)[case]
    acc = case % 2 == 0
    _check_fwbi_exact(_fwbi_case(cuda, B, sizes, E, seed=B + E, use_bias=use_bias, accumulate=acc), E, acc)


@pytest.mark.parametrize("E", PAD_E + [4, 16])
def test_field_wise_bi_nan_padding(cuda, E):
    B, sizes = 133, (2, 3, 1)
    _check_fwbi_exact(_fwbi_case(cuda, B, sizes, E, seed=E, accumulate=True), E, True)
    _nan_equals_zero_padding(lambda fill: _fwbi_case(cuda, B, sizes, E, seed=E, accumulate=True, fill=fill),
                             ("out", "dx", "dW"))


def test_field_wise_bi_c2_bench_shape(cuda):
    """tools/flen_bench.py's shape: 26 fields in groups i % 3, E = 32, B = 65536, dx added into the fields' columns.
    h and dx exactly; the weight gradients sum more terms than the exact range holds (the chunk tests pin them)."""
    r = _fwbi_case(cuda, 65536, (9, 9, 8), 32, seed=15, accumulate=True, offset=0)
    _check_fwbi_exact(r, 32, True, check_dw=False)


# ------------------------------------------------------------------------------------------------ CCPM
def _conv_stages(spec, C_in, gen, cuda, positive=False):
    """spec: ('conv', width, filters) / ('kmax', k) -> the kernel's stages, linear, with grid-valued kernels (1/2
    steps; ``positive``: 1/2 .. 3/2) and biases (1/4 steps)."""
    out, c = [], C_in
    for st in spec:
        if st[0] == "conv":
            _, w, f = st
            kern = _grid(gen, (w, 1, c, f), 1, 1, cuda).add_(1.0) if positive else _grid(gen, (w, 1, c, f), 3, 1, cuda)
            out.append(("conv", w, f, None, kern, _grid(gen, (f,), 3, 2, cuda)))
            c = f
        else:
            out.append(st)
    return out


def _conv_nblocks(stages, rows, E, C_in, cuda):
    """The CTA count of b2ctr_conv_stack_bwd (its partials), from its workspace function."""
    import ctypes
    from deepctr_b200 import kernels as K
    t = torch.zeros((1, 4096), device=cuda)
    a = K._conv_desc(stages, t, rows, E, C_in, 1, t)
    nw = sum(st[1] * st[4].shape[2] * st[2] + st[2] for st in stages if st[0] == "conv")

    def nblk(B):
        a.batch = B
        return _lib().b2ctr_conv_stack_bwd_workspace_bytes(ctypes.byref(a)) // (nw * 4)
    return nblk


def _conv_case(cuda, B, spec, rows, E, C_in, seed, accumulate=False, fill=None, distinct=False):
    """The stack on x at column 5 of a NaN-padded buffer, the output into a column window of a NaN buffer, dout read
    from a NaN-padded window, dx written (or added) into a window of a NaN buffer.  ``distinct``: every (sample, e)
    column of x holds distinct values, so a k-max after a positive width-1 convolution has no ties."""
    from deepctr_b200 import kernels as K
    gen = torch.Generator(device=cuda).manual_seed(seed)
    stages = _conv_stages(spec, C_in, gen, cuda, positive=distinct)
    k_out, c_out = K.conv_stack_check(rows, C_in, stages)
    w_in, w_out = rows * E * C_in, k_out * E * c_out
    xbuf = _padded((B + EXTRA_ROWS, 5 + w_in + 3), cuda, fill)
    if distinct:
        perm = torch.argsort(torch.rand((B, E * C_in, rows), generator=gen, device=cuda), dim=2)
        xv = (perm.float() - rows // 2).mul_(0.25).permute(0, 2, 1).reshape(B, w_in)
    else:
        xv = _grid(gen, (B, w_in), 1, 2, cuda)
    xbuf[:B, 5:5 + w_in] = xv
    x = xbuf[:B, 5:5 + w_in]
    out = Window(B, 2 + w_out + 6, 2, 1, w_out, w_out, cuda, fill)
    K.conv_stack_fwd(stages, x, rows, E, C_in, B, out.buf[:B, 2:2 + w_out])
    out.check_outside("conv_stack_fwd")
    dout = Window(B, 1 + w_out + 4, 1, 1, w_out, w_out, cuda, fill).fill(_grid(gen, (B, 1, w_out), 1, 2, cuda))
    dxw = Window(B, 3 + w_in + 2, 3, 1, w_in, w_in, cuda, fill)
    if accumulate:
        dxw.fill(_grid(gen, (B, 1, w_in), 3, 2, cuda))
    dx0 = dxw.values().clone()
    frozen = Frozen(xbuf, dout.buf)
    dws = K.conv_stack_bwd(stages, x, rows, E, C_in, B, dout.buf[:B, 1:1 + w_out], dx=dxw.buf[:B, 3:3 + w_in],
                           dx_accumulate=accumulate, want_dw=[st[0] == "conv" for st in stages])
    frozen.check("conv_stack_bwd")
    dxw.check_outside("conv_stack_bwd dx")
    weights = [w for st in stages if st[0] == "conv" for w in (st[4], st[5])]
    return dict(x=x, stages=stages, weights=weights, out=out.values(), g=dout.values(), dx=dxw.values(), dx0=dx0,
                dW=[w for d in dws if d is not None for w in d], shape=(rows, E, C_in))


def _check_conv_exact(r, accumulate, check_dw=True):
    rows, E, C_in = r["shape"]
    stages = r["stages"]

    def fn(x, *w):
        h, k = x.reshape(x.shape[0], rows, E, C_in), 0
        for st in stages:
            if st[0] == "conv":
                h, k = CO.conv2d(h, w[k], w[k + 1], None), k + 2
            else:
                h = CO.kmax(h, st[1], 1)
        return h
    dx = r["dx"].reshape(r["dx"].shape[0], -1)
    if accumulate:
        dx = dx - r["dx0"].reshape(dx.shape)
    # x (1/4) kernels (1/2) and biases (1/4) through two convolutions: 1/16; dx: dout (1/4) k k -> 1/16; dW: 1/32
    _exact_check(fn, r["x"], r["g"], r["weights"], (r["out"], dx, r["dW"]), (2.0 ** -4, 2.0 ** -4, 2.0 ** -5),
                 rows, E * C_in, "conv_stack", check_dw=check_dw)


CONV_SPEC = [("conv", 3, 2), ("conv", 2, 3)]           # rows 5, two input channels: 'same' padding both ways
KMAX_SPEC = [("conv", 1, 1), ("kmax", 3)]              # positive width-1 filter: the k-max sees x's order, no ties


@pytest.mark.parametrize("case", range(7), ids=["one", "below", "at", "above", "cap", "cap_plus_1", "c2_plus_1"])
@pytest.mark.parametrize("spec", ["conv", "kmax"])
def test_conv_stack_exact_at_block_boundaries(cuda, spec, case):
    """E = 1, so a CTA's 32 columns are 32 samples: B around one CTA, at the grid cap where the grid-stride loop
    starts to go round, and 65,537; the CTA count is the workspace's partial count."""
    gen = torch.Generator(device=cuda).manual_seed(0)
    sp, C_in = (CONV_SPEC, 2) if spec == "conv" else (KMAX_SPEC, 1)
    nblk = _conv_nblocks(_conv_stages(sp, C_in, gen, cuda), 5, 1, C_in, cuda)
    cap = nblk(1 << 24)
    assert nblk(31) == nblk(32) == 1 and nblk(33) == 2 and nblk(32 * cap) == nblk(32 * cap + 1) == cap
    B = [1, 31, 32, 33, 32 * cap, 32 * cap + 1, 65537][case]
    acc = case % 2 == 0
    _check_conv_exact(_conv_case(cuda, B, sp, 5, 1, C_in, seed=B, accumulate=acc, distinct=spec == "kmax"), acc)


@pytest.mark.parametrize("E", PAD_E + [4])
@pytest.mark.parametrize("spec", ["conv", "kmax"])
def test_conv_stack_nan_padding(cuda, spec, E):
    sp, C_in = (CONV_SPEC, 2) if spec == "conv" else (KMAX_SPEC, 1)
    B = 133

    def make(fill):
        return _conv_case(cuda, B, sp, 5, E, C_in, seed=E, accumulate=True, fill=fill, distinct=spec == "kmax")
    _check_conv_exact(make(None), True)
    _nan_equals_zero_padding(make, ("out", "dx", "dW"))


def test_conv_stack_equal_values_follow_the_tie_rule(cuda):
    """Equal values: the k-max keeps the lower rows (the reference's stable sort), exactly."""
    r = _conv_case(cuda, 257, [("kmax", 3)], 6, 2, 1, seed=3)
    _check_conv_exact(r, False)


def test_conv_stack_bench_shape(cuda):
    """tools/ccpm_bench.py's stack on 26 fields, E = 32, B = 65536: convolutions of widths 6 and 5 with 4 filters
    each, k-max 13 and 3, linear instead of tanh so the result is exact; ties resolved by the reference's rule.  The
    output and dx exactly; the weight gradients sum more terms than the exact range holds (the block tests pin
    them)."""
    spec = [("conv", 6, 4), ("kmax", CO.ccpm_k(1, 2, 26)), ("conv", 5, 4), ("kmax", 3)]
    _check_conv_exact(_conv_case(cuda, 65536, spec, 26, 32, 1, seed=16, accumulate=True), True, check_dw=False)
