"""GPU: the attention and field-weight kernels exactly, at their template, block and grid boundaries, with NaN in
every padding.

The operands are small integers (times a power of two), and every check first asserts, from the data, that the sum
of the absolute values of the terms of each result stays below 2^24 units of its grid, so every partial sum in every
order is exact in fp32.  The softmaxes are made exact too: every score is either its row's maximum or at least 128
below it, so expf gives exactly 1 or underflows to exactly 0 (the library builds without fast-math), the number of
maxima in a row is a power of two and every scale is a power of two.  The kernels must then equal the float64
restatements bit for bit: a dropped, doubled or misplaced sample, row, pair, round, warp, chunk or partial fails.
Inputs are windows of NaN-filled buffers (other columns, pitch gaps and the rows past the batch hold a NaN with a
payload), outputs, workspaces and saved state are written into windows of NaN-filled buffers, and nothing outside
them may change, bit for bit.

* b2ctr_mha_fwd / _bwd, exactly: d = 1 / 8 / 9 / 16 / 17 / 32 / 33 / 64 (DP = 8, 16, 32 and 64, padded and full)
  x T = 1 / 31 / 32 / 33 / 64 / 65 / 127 / 128 (one warp fewer or more per CTA), 2 heads, 6 samples, scale 2^7.
  Keys come in aligned pairs that are equal (a tie of two) or distinct; a marker coordinate, +-(2d - 1) in q and a
  distinct rank per key group in k, picks the extreme valid group of each query row, and the other coordinates
  (in [-1, 1]) can move no score across the 128 gap.  Four runs per shape: key and query lengths (0, 1, T - 1, T,
  random) with a residual; masks (an all-zero and an all-one row) with blinding; lengths with blinding and dropout
  0.5 (keep scale 2, the mask rebuilt from b2ctr_dropout) and a residual; masks with dropout.  Rows whose keys are
  all masked give every key 1/T: when T is not a power of two the reference reproduces that one fp32 rounding of
  1/T (and of the product and the residual sum) from exact intermediates, and dout keeps one row per such sample,
  so each dV entry is one rounded product.  out, dq, dk, dv, and the saved (max, sum) statistics;
* b2ctr_mha_* against the float64 restatement of test_bst_gpu with random data and the real scale 1/sqrt(d), at
  the same d x T grid, and at tools/bst_bench.py's shape (B = 8192, T = 50, 8 heads of 8), with tolerances;
* b2ctr_afm_fwd / _bwd, exactly: E = 1 / 4 / 5 / 8 / 9 / 16 / 17 / 32 x A = 1 / 2 / 3 / 4 / 5 / 8 / 9 / 16 (every
  EP and AP, padded and full) at F = 9 (36 pairs: a second round of 4); F = 2 / 3 / 8 / 9 / 64 (P = 1, 3, 28, 36,
  2016); batches from b2ctr_afm_bwd_workspace_bytes: 1, 3, 4, 5, around the backward's grid cap (528 CTAs of 4
  samples) and the forward's (1056 CTAs), and 65,537.  A +-1 / 0 marker column of x makes 1, 2 or 4 pairs tie at
  the top score 128 through attention unit 0 (W[0, 0] = 16, h[0] = 8); the other units have h = 0 and random W and
  bias, so dh is exercised on every AP lane.  The chosen pairs include the first and the last pair.  (The ds of
  tied pairs sum to 0, so dbias and dh[0] are 0 by construction here: the tolerance checks cover them.)  The
  workspace is NaN-filled, and W, bias and h are the leading part of NaN-filled allocations.  att, state, dx, dW,
  dbias and dh exactly, with no floor; tolerance checks with random data at the new E and A;
* b2ctr_senet_fwd / _bwd, exactly: E = 1 / 4 / 32 / 64 x F = 2 / 31 / 32 / 33 / 64 x R = 1 / 31 / 32 / 33 / 64;
  batches from b2ctr_senet_bwd_workspace_bytes: 1, 7, 8, 9, around the grid cap (528 CTAs of 8 warps) and 65,537;
  pre-activations that are exactly 0 (relu' = 0 there); V into a window of pitch wider than F*E; the saved (A1,
  A2) into a NaN buffer.  E = 5 / 33 with tolerances;
* b2ctr_fm_weighted_fwd / _bwd exactly at E = 1 / 31 / 32 / 33 / 64 / 65 (one to three 32-column chunks of dm),
  dx written, added to, or not asked for, dm asked for or not; b2ctr_field_scale_fwd / _bwd exactly at E = 1 / 2 /
  3 / 5 / 9 / 17 / 33 (group widths 1 to 32) with B*F not a multiple of the groups per warp;
  b2ctr_softmax_rows_fwd / _bwd exactly at 1 / 31 / 32 / 33 / 64 / 100 columns with scale 1 and IFM's 26 (26/n is
  exact for n a power of two).  Every one at a batch past its grid cap; tolerance checks with random data at the
  same shapes.
"""
import ctypes as C

import pytest
import torch

from test_bst_gpu import _close, _mha_case
from test_fibinet_gpu import _check_senet
from test_ifm_gpu import _check_fm, _check_scale
from test_pairwise_gpu import _check_afm
from test_product_kernels_exact_gpu import NAN_BITS, Frozen, Window, _fits, _lib, _nan_like, _same

pytestmark = pytest.mark.gpu

GAP = 128.0                              # expf(-128) underflows to exactly 0 in fp32
PAD_SCORE = -4294967296.0                # the kernel's masked score, -2^32 + 1 rounded to fp32
NUM_SMS = 132                            # grid_for's SM count: caps are NUM_SMS * blocks per SM


def _kern():
    from deepctr_b200 import kernels as K
    return K


def _ints(gen, shape, lo, hi):
    """Integers in [lo, hi] as fp32, drawn on the host so the cases are the same on every device."""
    return torch.randint(lo, hi + 1, tuple(shape), generator=gen).to(torch.float32)


def _check(status, what):
    from deepctr_b200 import _lib as L
    L.check(status, what)


def _round32(t):
    return t.float().double()


class Flat:
    """A contiguous output of n floats at the front of a NaN buffer with a NaN tail."""

    def __init__(self, n, device, tail=9):
        self.n = n
        self.buf = _nan_like((n + tail,), device)

    def values(self):
        return self.buf[:self.n]

    def check_outside(self, what):
        tail = self.buf[self.n:].view(torch.int32)
        assert bool((tail == NAN_BITS).all()), "%s: the NaN tail behind the output was written" % what


def _put(B, ld, col0, vals, device):
    """A Window of a NaN buffer holding vals [B, width] at column col0."""
    w = Window(B, ld, col0, 1, vals.shape[1], vals.shape[1], device)
    return w.fill(vals.to(device).reshape(B, 1, -1))


def _nan_workspace(nbytes, device):
    return _nan_like((max(nbytes, 4) // 4 + 9,), device)


def _pow2(n):
    return (n > 0) & ((n & (n - 1)) == 0)


def _exact_softmax(s, what, valid=None):
    """Weights of a softmax whose scores are exact: every score is its row's maximum or at least GAP below it.
    -> (weights with 1/n on the n maxima, n).  Rows with no valid entry (``valid`` all False) may have any n."""
    M = s.max(-1, keepdim=True).values
    win = s == M
    assert bool((win | (s <= M - GAP)).all()), "%s: a score is neither its row's maximum nor %g below it" % (what, GAP)
    n = win.sum(-1, keepdim=True)
    ok = _pow2(n) if valid is None else _pow2(n) | ~valid.any(-1, keepdim=True)
    assert bool(ok.all()), "%s: a row's number of maxima is not a power of two" % what
    return win.double() / n.double(), n, M


# ================================================================================================ MHA
MHA_D = [1, 8, 9, 16, 17, 32, 33, 64]
MHA_T = [1, 31, 32, 33, 64, 65, 127, 128]
MHA_HEADS = 2
MHA_B = 6
MHA_SCALE = 128.0
# (validity kind, blinding, dropout rate, residual)
MHA_RUNS = {"len_res": ("len", False, 0.0, True), "mask_blind": ("mask", True, 0.0, False),
            "len_blind_drop_res": ("len", True, 0.5, True), "mask_drop": ("mask", False, 0.5, False)}


def _mha_valid(kind, B, T, gen):
    """int32 lengths [B] (0, 1, T - 1, T, then random) or uint8 masks [B, T] (all zero, all one, random)."""
    if kind == "len":
        ln = torch.randint(0, T + 1, (B,), generator=gen, dtype=torch.int32)
        ln[:4] = torch.tensor([0, 1, T - 1, T], dtype=torch.int32)
        return ln, torch.arange(T)[None, :] < ln[:, None].long()
    m = (torch.rand((B, T), generator=gen) < 0.6).to(torch.uint8)
    m[0], m[1] = 0, 1
    return m, m.bool()


def _mha_operands(gen, B, T, H, d):
    """q, k, v, residual, dout [B, T, H, d] (host).  Keys in aligned pairs, equal or distinct; k[..., 0] a distinct
    rank per key group, q[..., 0] = +-(2d - 1): the q.k of two groups differ by at least 1 (128 after the scale)."""
    k = _ints(gen, (B, T, H, d), -1, 1)
    rank = torch.argsort(torch.rand((B, T, H), generator=gen), dim=1).to(torch.float32)
    k[..., 0] = rank - T // 2
    paired = torch.rand((B, T // 2, H), generator=gen) < 0.5
    odd = k[:, 1:2 * (T // 2):2]
    odd[paired] = k[:, 0:2 * (T // 2):2][paired]          # the pair's second key repeats the first
    q = _ints(gen, (B, T, H, d), -1, 1)
    sign = torch.randint(0, 2, (B, T, H), generator=gen).to(torch.float32) * 2 - 1
    q[..., 0] = sign * (2 * d - 1)
    v, res, dout = (_ints(gen, (B, T, H, d), -1, 1) for _ in range(3))
    return q, k, v, res, dout


def _mha_reference(q, k, v, res, dout, qvalid, kvalid, blinding, drop, scale):
    """float64 restatement with the exact softmax; all tensors [B, T, H, d] on the device, qvalid / kvalid bool
    [B, T], drop [B, H, T, T] or None.  -> dict of out, dq, dk, dv [B*T, H*d], stats [B, H, T, 2] and the bounds."""
    B, T, H, d = q.shape
    Q, K_, V, G = (t.double().permute(0, 2, 1, 3) for t in (q, k, v, dout))        # [B, H, T, d]
    eye = torch.eye(T, dtype=torch.bool, device=q.device)
    valid = kvalid[:, None, None, :].expand(B, H, T, T)
    if blinding:
        valid = valid & ~eye
    S = torch.where(valid, (Q @ K_.transpose(-1, -2)) * scale, torch.full((), PAD_SCORE, device=q.device,
                                                                                 dtype=torch.float64))
    p, n, M = _exact_softmax(S, "mha scores", valid)
    # a row with no valid key: every key gets 1/T, rounded once to fp32 when T is not a power of two
    p = torch.where(_pow2(n), p, _round32(p))
    qm = qvalid[:, None, :, None].double()
    P = p * qm * (drop if drop is not None else 1.0)
    O = P @ V
    gv = G @ V.transpose(-1, -2)
    D = (P * gv).sum(-1, keepdim=True)
    dS = torch.where(valid, p * (gv * qm * (drop if drop is not None else 1.0) - D), torch.zeros((), device=q.device,
                                                                                                  dtype=torch.float64))
    flat = lambda t: t.permute(0, 2, 1, 3).reshape(B * T, H * d)                  # noqa: E731
    out = _round32(flat(O))
    if res is not None:
        out = _round32(out + res.double().reshape(B * T, H * d))
    r = dict(out=out, dq=flat(dS @ K_) * scale, dk=flat(dS.transpose(-1, -2) @ Q) * scale,
             dv=_round32(flat(P.transpose(-1, -2) @ G)), stats=torch.stack([M[..., 0], n[..., 0].double()], -1))
    aP, adS = P.abs(), dS.abs()
    r["bounds"] = dict(out=flat(aP @ V.abs()) + (res.double().abs().reshape(B * T, H * d) if res is not None else 0),
                       dq=flat(adS @ K_.abs()), dk=flat(adS.transpose(-1, -2) @ Q.abs()),
                       dv=flat(aP.transpose(-1, -2) @ G.abs()),
                       D=(aP * (G.abs() @ V.abs().transpose(-1, -2))).sum(-1))
    return r


def _mha_exact_case(cuda, B, T, d, run, seed):
    from deepctr_b200 import _lib as L
    K = _kern()
    kind, blinding, rate, use_res = MHA_RUNS[run]
    H, W = MHA_HEADS, MHA_HEADS * d
    gen = torch.Generator().manual_seed(seed)
    q, k, v, res, dout = _mha_operands(gen, B, T, H, d)
    qv, qvalid = _mha_valid(kind, B, T, gen)
    kv, kvalid = _mha_valid(kind, B, T, gen)
    # samples with a query row that sees no key: when T is not a power of two, dout keeps one row there
    eye = torch.eye(T, dtype=torch.bool)
    seen = kvalid[:, None, :] & ~eye if blinding else kvalid[:, None, :].expand(B, T, T)
    if T & (T - 1):
        for b in torch.nonzero((~seen.any(-1)).any(-1)).flatten().tolist():
            keep = b % T
            dout[b, :keep] = 0
            dout[b, keep + 1:] = 0
    # q / k / v / residual are windows of one NaN buffer, dout of another
    ld = 4 * W + 9
    rows = B * T
    src = Window(rows, ld, 0, 4, W, W + 2, cuda)
    src.fill(torch.stack([t.reshape(rows, W) for t in (q, k, v, res)], 1).to(cuda))
    blocks = src.values()
    qw, kw, vw, rw = (blocks[:, i] for i in range(4))
    gwin = _put(rows, W + 5, 2, dout.reshape(rows, W), cuda)
    gw = gwin.values()[:, 0]
    stats = Flat(B * H * T * 2, cuda)
    out = Window(rows, W + 7, 3, 1, W, W, cuda)
    qv, kv = qv.to(cuda), kv.to(cuda)
    lens = dict(qlen=qv, klen=kv, qmask=None, kmask=None) if kind == "len" else \
        dict(qlen=None, klen=None, qmask=qv, kmask=kv)
    a = K._mha_desc(qw, ld, kw, ld, vw, ld, B, T, H, d, MHA_SCALE, blinding, rate, seed, stats.values(), **lens)
    a.res, a.ldr = (rw.data_ptr(), ld) if use_res else (None, 0)
    a.out, a.ldo = out.buf[:, 3:].data_ptr(), out.ld
    frozen = Frozen(src.buf, gwin.buf)
    L.check(_lib().b2ctr_mha_fwd(C.byref(a), K.stream()), "mha_fwd")
    out.check_outside("mha_fwd out")
    stats.check_outside("mha_fwd stats")
    grads = [Window(rows, W + 3 + i, 1 + i, 1, W, W, cuda) for i in range(3)]
    a.dout, a.lddo = gw.data_ptr(), gwin.ld
    (a.dq, a.lddq), (a.dk, a.lddk), (a.dv, a.lddv) = [(g.buf[:, 1 + i:].data_ptr(), g.ld) for i, g in enumerate(grads)]
    stats_before = stats.buf.clone()
    L.check(_lib().b2ctr_mha_bwd(C.byref(a), K.stream()), "mha_bwd")
    frozen.check("mha_bwd")
    assert torch.equal(stats.buf.view(torch.int32), stats_before.view(torch.int32)), "mha_bwd wrote its statistics"
    for g, name in zip(grads, ("dq", "dk", "dv")):
        g.check_outside("mha_bwd " + name)
    drop = None
    if rate:
        ones = torch.ones((H * B, T, T), dtype=torch.float32, device=cuda)
        drop = K.dropout(ones, rate, seed).double().reshape(H, B, T, T).transpose(0, 1)
    ref = _mha_reference(*(t.to(cuda) for t in (q, k, v)), res.to(cuda) if use_res else None, dout.to(cuda),
                         qvalid.to(cuda), kvalid.to(cuda), blinding, drop, MHA_SCALE)
    # grids: P in 1/128 (1/T on a row that sees no key, else 1/2) times integers; ds in 1/4 (0 on a row that sees
    # no key), dq / dk = 2^7 * ds * integers
    bd = ref["bounds"]
    for name, unit in (("out", 1.0 / 128), ("dv", 1.0 / 128), ("D", 1.0 / 128), ("dq", 32.0), ("dk", 32.0)):
        _fits(bd[name], unit, "mha " + name)
    _same(out.values().reshape(rows, W), ref["out"], "mha out")
    _same(stats.values().reshape(B, H, T, 2), ref["stats"], "mha stats")
    for g, name in zip(grads, ("dq", "dk", "dv")):
        _same(g.values().reshape(rows, W), ref[name], "mha " + name)


@pytest.mark.parametrize("run", sorted(MHA_RUNS))
@pytest.mark.parametrize("T", MHA_T)
@pytest.mark.parametrize("d", MHA_D)
def test_mha_exact(cuda, d, T, run):
    _mha_exact_case(cuda, MHA_B, T, d, run, seed=1000 * d + T + len(run))


@pytest.mark.parametrize("T", MHA_T)
@pytest.mark.parametrize("d", MHA_D)
def test_mha_random_data_within_tolerance(cuda, d, T):
    """Random normal data, the real scale 1/sqrt(d); lengths with blinding on odd T, masks without on even T."""
    out, (dq, dk, dv), ref, ts, _ = _mha_case(cuda, 13, T, MHA_HEADS * d, MHA_HEADS, bool(T % 2),
                                              "len" if T % 2 else "mask", seed_np=d + T)
    _close(out, ref, "out")
    _close(dq, ts[0].grad, "dq")
    _close(dk, ts[1].grad, "dk")
    _close(dv, ts[2].grad, "dv")


def test_mha_bst_bench_shape_within_tolerance(cuda):
    """tools/bst_bench.py's attention: B = 8192, T = 50, E = 64 in 8 heads of 8, lengths, a residual."""
    out, (dq, dk, dv), ref, ts, _ = _mha_case(cuda, 8192, 50, 64, 8, False, "len", seed_np=5)
    _close(out, ref, "out")
    _close(dq, ts[0].grad, "dq")
    _close(dk, ts[1].grad, "dk")
    _close(dv, ts[2].grad, "dv")


# ================================================================================================ AFM
AFM_E = [1, 4, 5, 8, 9, 16, 17, 32]
AFM_A = [1, 2, 3, 4, 5, 8, 9, 16]
AFM_W00, AFM_H0 = 16.0, 8.0              # attention unit 0: a top pair scores 8 * relu(16) = 128, the others 0
AFM_TOP = AFM_W00 * AFM_H0


def _afm_nblk(E, A):
    L = _lib()
    EP = 4 if E <= 4 else 8 if E <= 8 else 16 if E <= 16 else 32
    AP = 1 if A <= 1 else 2 if A <= 2 else 4 if A <= 4 else 8 if A <= 8 else 16
    return lambda B: L.b2ctr_afm_bwd_workspace_bytes(E, A, B) // ((EP * AP + 2 * AP) * 4)


def _afm_batches(E, A):
    """1, 3, 4, 5 (a CTA takes 4 samples), around the backward's grid cap (the workspace's CTA count) and the
    forward's (grid_for(B, 4, 8): twice the backward's CTAs), and 65,537."""
    nb = _afm_nblk(E, A)
    cap = nb(1 << 30)
    assert nb(4) == 1 and nb(5) == 2 and cap == NUM_SMS * 4 and nb(4 * cap - 1) == nb(4 * cap + 1) == cap
    fwd = 2 * cap * 4
    return [1, 3, 4, 5, 4 * cap - 1, 4 * cap, 4 * cap + 1, fwd - 1, fwd, fwd + 1, 65537]


AFM_BATCH_IDS = ["one", "three", "cta", "cta_plus_1", "bwd_cap_minus_1", "bwd_cap", "bwd_cap_plus_1",
                 "fwd_cap_minus_1", "fwd_cap", "fwd_cap_plus_1", "c2_plus_1"]


def _afm_operands(gen, B, F, E, A):
    """x [B, F, E]: column 0 a +-1 / 0 marker, the others integers in [-1, 1].  Samples cycle through ties of 1, 2
    and 4 top pairs (two +1 fields and one -1; two and two; three and two), as many as F allows; every 4th sample
    puts its +1 pair on the last two fields (the last pair), every 4th other one on the first two."""
    x = _ints(gen, (B, F, E), -1, 1)
    x[:, :, 0] = 0
    key = torch.rand((B, F), generator=gen)
    key[1::4, F - 2:] = -1.0
    key[3::4, :2] = -1.0
    perm = torch.argsort(key, dim=1)
    kinds = [(2, min(F - 2, 1))] + ([(2, 2)] if F >= 4 else []) + ([(3, 2)] if F >= 5 else [])
    for c, (npos, nneg) in enumerate(kinds):
        sl = slice(c, B, len(kinds))
        xs = x[sl]
        xs.scatter_(1, perm[sl, :npos, None].expand(-1, -1, 1), 1.0)            # marker column is column 0
        if nneg:
            xs.scatter_(1, perm[sl, npos:npos + nneg, None].expand(-1, -1, 1), -1.0)
        x[sl] = xs
    W = _ints(gen, (E, A), 0, 1) * 2 - 1                                  # +-1: no unit is constant
    W[:, 0] = 0
    W[0, 0] = AFM_W00
    bias = _ints(gen, (A,), -1, 1)
    bias[0] = 0
    h = torch.zeros(A)
    h[0] = AFM_H0
    g = _ints(gen, (B, E), -1, 1)
    return x, W, bias, h, g


def _afm_reference(x, W, bias, h, g, visit, rows):
    """float64 AFMLayer with the exact softmax, over sample chunks: visit(slice, att, dx, abs-bounds) and returns
    (dW, dbias, dh) and their abs-bounds."""
    B, F, E = x.shape
    i, j = torch.triu_indices(F, F, 1, device=x.device)
    W64, b64, h64 = W.double(), bias.double(), h.double()
    acc = [0.0] * 6
    for b0 in range(0, B, rows):
        sl = slice(b0, min(B, b0 + rows))
        xs, gs = x[sl].double(), g[sl].double()
        prod = xs[:, i] * xs[:, j]                                          # [n, P, E]
        t = prod @ W64 + b64                                                # [n, P, A]
        s = torch.relu(t) @ h64                                             # [n, P]
        alpha, _, _ = _exact_softmax(s, "afm scores")
        att = (alpha[..., None] * prod).sum(1)
        gp = prod @ gs[:, :, None]
        ds = alpha * (gp[..., 0] - (att * gs).sum(1, keepdim=True))         # [n, P]
        dt = ds[..., None] * h64 * (t > 0)
        dprod = alpha[..., None] * gs[:, None, :] + dt @ W64.T
        dx = torch.zeros_like(xs)
        dx.index_add_(1, i, dprod * xs[:, j]).index_add_(1, j, dprod * xs[:, i])
        aprod, ads, adt = prod.abs(), ds.abs(), dt.abs()
        adprod = alpha[..., None] * gs.abs()[:, None, :] + adt @ W64.abs().T
        adx = torch.zeros_like(xs)
        adx.index_add_(1, i, adprod * xs[:, j].abs()).index_add_(1, j, adprod * xs[:, i].abs())
        visit(sl, att, dx, dict(att=(alpha[..., None] * aprod).sum(1), dx=adx,
                                t=aprod @ W64.abs() + b64.abs(), gp=aprod @ gs.abs()[:, :, None]))
        parts = [torch.einsum("npe,npa->ea", prod, dt), dt.sum((0, 1)), (ds[..., None] * torch.relu(t)).sum((0, 1)),
                 torch.einsum("npe,npa->ea", aprod, adt), adt.sum((0, 1)), (ads[..., None] * torch.relu(t)).sum((0, 1))]
        acc = [a + p for a, p in zip(acc, parts)]
    return acc[:3], acc[3:]


def _afm_exact_case(cuda, B, F, E, A, seed):
    K = _kern()
    L = _lib()
    gen = torch.Generator().manual_seed(seed)
    x, W, bias, h, g = _afm_operands(gen, B, F, E, A)
    xw = _put(B, F * E + 7, 3, x.reshape(B, F * E), cuda)
    xv, ldx = xw.values()[:, 0], xw.ld
    Wf, bf, hf = Flat(E * A, cuda), Flat(A, cuda), Flat(A, cuda)
    Wf.values()[:] = W.reshape(-1).to(cuda)
    bf.values()[:] = bias.to(cuda)
    hf.values()[:] = h.to(cuda)
    att = Window(B, E + 5, 2, 1, E, E, cuda)
    state = Flat(2 * B, cuda)
    frozen = Frozen(xw.buf, Wf.buf, bf.buf, hf.buf)
    _check(L.b2ctr_afm_fwd(xv.data_ptr(), ldx, F, E, A, Wf.buf.data_ptr(), bf.buf.data_ptr(), hf.buf.data_ptr(),
                           att.buf[:, 2:].data_ptr(), att.ld, state.buf.data_ptr(), B, K.stream()), "afm_fwd")
    att.check_outside("afm_fwd att")
    state.check_outside("afm_fwd state")
    gw = _put(B, E + 4, 1, g, cuda)
    dx = Window(B, F * E + 6, 4, 1, F * E, F * E, cuda)
    dW, db, dh = Flat(E * A, cuda), Flat(A, cuda), Flat(A, cuda)
    nbytes = L.b2ctr_afm_bwd_workspace_bytes(E, A, B)
    ws = _nan_workspace(nbytes, cuda)
    frozen_bwd = Frozen(gw.buf, att.buf, state.buf)
    _check(L.b2ctr_afm_bwd(gw.buf[:, 1:].data_ptr(), gw.ld, xv.data_ptr(), ldx, F, E, A, Wf.buf.data_ptr(),
                           bf.buf.data_ptr(), hf.buf.data_ptr(), state.buf.data_ptr(), att.buf[:, 2:].data_ptr(),
                           att.ld, dx.buf[:, 4:].data_ptr(), dx.ld, dW.buf.data_ptr(), db.buf.data_ptr(),
                           dh.buf.data_ptr(), B, ws.data_ptr(), nbytes, K.stream()), "afm_bwd")
    frozen.check("afm")
    frozen_bwd.check("afm_bwd")
    dx.check_outside("afm_bwd dx")
    for o, n in ((dW, "dW"), (db, "dbias"), (dh, "dh")):
        o.check_outside("afm_bwd " + n)
    # grids: prod, t, g integers; alpha in 1/4; att in 1/4, ds and everything after it in 1/16
    got_att, got_dx = att.values().reshape(B, E), dx.values().reshape(B, F, E)
    got_state = state.values().reshape(B, 2)

    def visit(sl, a, d, bd):
        _fits(bd["att"], 0.25, "afm att")
        _fits(bd["dx"], 1.0 / 16, "afm dx")
        _fits(bd["t"], 1.0, "afm t")
        _fits(bd["gp"], 1.0, "afm <g, prod>")
        _same(got_att[sl], a, "afm att")
        _same(got_dx[sl], d, "afm dx")
        top = got_state[sl, 0]
        assert bool(((top == AFM_TOP) | (top == 0)).all()), "afm state: the maximum is not an exact score"
    rows = max(1, (1 << 22) // (F * (F - 1) // 2 * max(E, A)))
    (rW, rb, rh), (aW, ab, ah) = _afm_reference(x.to(cuda), W.to(cuda), bias.to(cuda), h.to(cuda), g.to(cuda),
                                                visit, rows)
    for bnd, n in ((aW, "dW"), (ab, "dbias"), (ah, "dh")):
        _fits(bnd, 1.0 / 16, "afm " + n)
    _same(dW.values().reshape(E, A), rW, "afm dW")
    _same(db.values(), rb, "afm dbias")
    _same(dh.values(), rh, "afm dh")


@pytest.mark.parametrize("A", AFM_A)
@pytest.mark.parametrize("E", AFM_E)
def test_afm_exact_every_template_size(cuda, E, A):
    """F = 9: 36 pairs, a second round of 4; B = 13, four CTAs, the last one short."""
    _afm_exact_case(cuda, 13, 9, E, A, seed=100 * E + A)


@pytest.mark.parametrize("E,A", [(5, 3), (32, 16), (1, 2)])
@pytest.mark.parametrize("F", [2, 3, 8, 9, 64])
def test_afm_exact_pair_rounds(cuda, F, E, A):
    """P = 1, 3, 28 (fewer pairs than lanes), 36 (a second round of 4) and 2016 (63 rounds)."""
    _afm_exact_case(cuda, 37, F, E, A, seed=7 * F + E + A)


@pytest.mark.parametrize("case", range(len(AFM_BATCH_IDS)), ids=AFM_BATCH_IDS)
@pytest.mark.parametrize("F,E,A", [(9, 5, 3), (64, 4, 2)], ids=["F9_E5_A3", "F64_E4_A2"])
def test_afm_exact_at_block_and_grid_boundaries(cuda, F, E, A, case):
    B = _afm_batches(E, A)[case]
    _afm_exact_case(cuda, B, F, E, A, seed=B + F)


@pytest.mark.parametrize("F,E,A", [(9, 1, 2), (26, 9, 2), (9, 17, 5), (64, 16, 9), (3, 32, 16)])
def test_afm_random_data_within_tolerance(cuda, F, E, A):
    _check_afm(cuda, 1001, F, E, A, 5, F + E + A)


# ================================================================================================ SENET
SENET_E = [1, 4, 32, 64]
SENET_F = [2, 31, 32, 33, 64]
SENET_R = [1, 31, 32, 33, 64]


def _senet_batches(F, R):
    """1, 7, 8, 9 (a CTA takes 8 samples per lockstep round), around the grid cap (the workspace's CTA count) and
    65,537."""
    L = _lib()
    nb = lambda B: L.b2ctr_senet_bwd_workspace_bytes(F, R, B) // (2 * F * R * 4)      # noqa: E731
    cap = nb(1 << 30)
    assert nb(8) == 1 and nb(9) == 2 and cap == NUM_SMS * 4 and nb(8 * cap - 1) == nb(8 * cap + 1) == cap
    return [1, 7, 8, 9, 8 * cap - 1, 8 * cap, 8 * cap + 1, 65537]


SENET_BATCH_IDS = ["one", "seven", "cta", "cta_plus_1", "cap_minus_1", "cap", "cap_plus_1", "c2_plus_1"]


def _senet_reference(x, W1, W2, g, E):
    """float64 SENETLayer and its backward (relu' = 0 at 0), x / g [B, F, E] -> dict with the abs-bounds."""
    x, g, W1, W2 = x.double(), g.double(), W1.double(), W2.double()
    Z = x.sum(-1) / E
    t1 = Z @ W1
    A1 = torch.relu(t1)
    t2 = A1 @ W2
    A2 = torch.relu(t2)
    d2 = (A2 > 0) * (g * x).sum(-1)
    d1 = (A1 > 0) * (d2 @ W2.T)
    dZ = d1 @ W1.T
    r = dict(V=x * A2[..., None], dx=g * A2[..., None] + (dZ / E)[..., None], dW1=Z.T @ d1, dW2=A1.T @ d2, t1=t1, t2=t2,
             saved=torch.cat([A1, A2], 1))
    aZ, aA1, ad2 = Z.abs(), (Z.abs() @ W1.abs()), (g * x).abs().sum(-1)
    ad1 = ad2 @ W2.abs().T
    r["bounds"] = dict(A1=aA1, A2=aA1 @ W2.abs(), dx=g.abs() * (aA1 @ W2.abs())[..., None] + (ad1 @ W1.abs().T)[..., None],
                       dW1=aZ.T @ ad1, dW2=aA1.T @ ad2)
    return r


def _senet_exact_case(cuda, B, F, E, R, seed, zero_preact=False):
    K = _kern()
    L = _lib()
    gen = torch.Generator().manual_seed(seed)
    x, g = _ints(gen, (B, F * E), -1, 1), _ints(gen, (B, F * E), -1, 1)
    W1, W2 = _ints(gen, (F, R), -1, 1), _ints(gen, (R, F), -1, 1)
    if zero_preact:                      # unit 0 and field 0 get a pre-activation of exactly 0 in every sample
        W1[:, 0] = 0
        W2[:, 0] = 0
    xw = _put(B, F * E + 5, 2, x, cuda)
    v = Window(B, F * E + 11, 4, 1, F * E, F * E, cuda)           # pitch wider than F * E
    saved = Flat(B * (R + F), cuda)
    W1d, W2d = W1.to(cuda), W2.to(cuda)
    frozen = Frozen(xw.buf, W1d, W2d)
    _check(L.b2ctr_senet_fwd(xw.buf[:, 2:].data_ptr(), xw.ld, F, E, R, W1d.data_ptr(), W2d.data_ptr(),
                             v.buf[:, 4:].data_ptr(), v.ld, saved.buf.data_ptr(), B, K.stream()), "senet_fwd")
    v.check_outside("senet_fwd V")
    saved.check_outside("senet_fwd saved")
    gw = _put(B, F * E + 3, 3, g, cuda)
    dx = Window(B, F * E + 2, 1, 1, F * E, F * E, cuda)
    dW1, dW2 = Flat(F * R, cuda), Flat(R * F, cuda)
    nbytes = L.b2ctr_senet_bwd_workspace_bytes(F, R, B)
    ws = _nan_workspace(nbytes, cuda)
    frozen_bwd = Frozen(gw.buf, saved.buf)
    _check(L.b2ctr_senet_bwd(gw.buf[:, 3:].data_ptr(), gw.ld, xw.buf[:, 2:].data_ptr(), xw.ld, F, E, R,
                             W1d.data_ptr(), W2d.data_ptr(), saved.buf.data_ptr(), dx.buf[:, 1:].data_ptr(), dx.ld,
                             dW1.buf.data_ptr(), dW2.buf.data_ptr(), B, ws.data_ptr(), nbytes, K.stream()),
           "senet_bwd")
    frozen.check("senet")
    frozen_bwd.check("senet_bwd")
    dx.check_outside("senet_bwd dx")
    dW1.check_outside("senet_bwd dW1")
    dW2.check_outside("senet_bwd dW2")
    ref = _senet_reference(x.to(cuda).reshape(B, F, E), W1d, W2d, g.to(cuda).reshape(B, F, E), E)
    # grids: Z, A1, A2, V and dx in 1/E, d2 / d1 / dZ integers, dW1 / dW2 in 1/E
    u = 1.0 / E
    for n in ("A1", "A2", "dx", "dW1", "dW2"):
        _fits(ref["bounds"][n], u, "senet " + n)
    _same(v.values().reshape(B, F, E), ref["V"], "senet V")
    _same(saved.values().reshape(B, R + F), ref["saved"], "senet saved")
    _same(dx.values().reshape(B, F, E), ref["dx"], "senet dx")
    _same(dW1.values().reshape(F, R), ref["dW1"], "senet dW1")
    _same(dW2.values().reshape(R, F), ref["dW2"], "senet dW2")
    return ref


@pytest.mark.parametrize("R", SENET_R)
@pytest.mark.parametrize("F", SENET_F)
@pytest.mark.parametrize("E", SENET_E)
def test_senet_exact_shapes(cuda, E, F, R):
    """E = 64: the mean and <g, x> are two-chunk warp sums; F and R on both sides of a warp; B = 11: a full
    lockstep round and a round of 3."""
    _senet_exact_case(cuda, 11, F, E, R, seed=E * 10000 + F * 100 + R)


@pytest.mark.parametrize("case", range(len(SENET_BATCH_IDS)), ids=SENET_BATCH_IDS)
@pytest.mark.parametrize("F,E,R", [(3, 4, 2), (33, 1, 31)], ids=["F3_E4_R2", "F33_E1_R31"])
def test_senet_exact_at_round_and_grid_boundaries(cuda, F, E, R, case):
    B = _senet_batches(F, R)[case]
    _senet_exact_case(cuda, B, F, E, R, seed=B + F)


@pytest.mark.parametrize("E", [4, 64])
def test_senet_relu_gradient_at_zero(cuda, E):
    """A zero column of W1 and of W2: a pre-activation of exactly 0 in every sample, where relu' is 0."""
    ref = _senet_exact_case(cuda, 133, 7, E, 5, seed=E, zero_preact=True)
    assert bool((ref["t1"][:, 0] == 0).all()) and bool((ref["t2"][:, 0] == 0).all())


@pytest.mark.parametrize("F,R", [(2, 1), (31, 33), (33, 31), (64, 64)])
@pytest.mark.parametrize("E", [5, 33])
def test_senet_random_data_within_tolerance(cuda, E, F, R):
    _check_senet(cuda, 1001, F, E, R, E + F + R)


# ================================================================================================ IFM / DIFM
ROW_WARPS_CAP = NUM_SMS * 8 * 8          # grid_for(B, 8, 8): 1056 CTAs of 8 warps, one row (sample) per warp
FMW_E = [1, 31, 32, 33, 64, 65]
WANTS = ["both", "dx", "dm"]


def _fm_weighted_case(cuda, B, F, E, acc, want, seed):
    L, K = _lib(), _kern()
    gen = torch.Generator().manual_seed(seed)
    x = _ints(gen, (B, F * E), -2, 2) * 0.5
    m = _ints(gen, (B, F), -2, 2)
    g = _ints(gen, (B,), -2, 2)
    xw, mw = _put(B, F * E + 5, 3, x, cuda), _put(B, F + 4, 1, m, cuda)
    gf = Flat(B, cuda)
    gf.values()[:] = g.to(cuda)
    out = Flat(B, cuda)
    frozen = Frozen(xw.buf, mw.buf, gf.buf)
    xp, mp = xw.buf[:, 3:].data_ptr(), mw.buf[:, 1:].data_ptr()
    _check(L.b2ctr_fm_weighted_fwd(xp, xw.ld, mp, mw.ld, F, E, out.buf.data_ptr(), B, K.stream()), "fm_weighted_fwd")
    out.check_outside("fm_weighted_fwd")
    dx = Window(B, F * E + 4, 2, 1, F * E, F * E, cuda)
    if acc:
        dx.fill(_ints(gen, (B, 1, F * E), -3, 3).to(cuda))
    dx0 = dx.values().clone()
    dm = Window(B, F + 3, 1, 1, F, F, cuda)
    _check(L.b2ctr_fm_weighted_bwd(xp, xw.ld, mp, mw.ld, F, E, gf.buf.data_ptr(),
                                   dx.buf[:, 2:].data_ptr() if want != "dm" else None, dx.ld, int(acc),
                                   dm.buf[:, 1:].data_ptr() if want != "dx" else None, dm.ld, B, K.stream()),
           "fm_weighted_bwd")
    frozen.check("fm_weighted")
    dx.check_outside("fm_weighted_bwd dx")
    dm.check_outside("fm_weighted_bwd dm")
    x64, m64, g64 = x.to(cuda).double().reshape(B, F, E), m.to(cuda).double(), g.to(cuda).double()
    v = x64 * m64[..., None]
    S = v.sum(1, keepdim=True)
    r = S - v
    aS = v.abs().sum(1, keepdim=True)
    # grids: v in 1/2, out 0.5 (S^2 - q) in 1/8, dx = g m (S - m x) in 1/2, dm = g sum_e x (S - m x) in 1/4
    _fits(0.5 * (aS * aS + v * v).sum((1, 2)), 0.125, "fm_weighted out")
    _fits(g64.abs()[:, None, None] * m64.abs()[..., None] * (aS + v.abs()) +
          (dx0.abs().double().reshape(B, F, E) if acc else 0), 0.5, "fm_weighted dx")
    _fits(g64.abs()[:, None] * (x64.abs() * (aS + v.abs())).sum(2), 0.25, "fm_weighted dm")
    _same(out.values(), 0.5 * (S[:, 0] ** 2 - (v * v).sum(1)).sum(1), "fm_weighted out")
    if want != "dm":
        want_dx = g64[:, None, None] * m64[..., None] * r + (dx0.double().reshape(B, F, E) if acc else 0)
        _same(dx.values().reshape(B, F, E), want_dx, "fm_weighted dx")
    else:
        assert torch.equal(dx.values().view(torch.int32), dx0.view(torch.int32)), "fm_weighted_bwd wrote dx"
    if want != "dx":
        _same(dm.values().reshape(B, F), g64[:, None] * (x64 * r).sum(2), "fm_weighted dm")
    else:
        assert bool((dm.values().view(torch.int32) == NAN_BITS).all()), "fm_weighted_bwd wrote dm"


@pytest.mark.parametrize("want", WANTS)
@pytest.mark.parametrize("acc", [False, True], ids=["write", "accumulate"])
@pytest.mark.parametrize("E", FMW_E)
def test_fm_weighted_exact_past_the_grid_cap(cuda, E, acc, want):
    """F = 7, B = 13 past the cap of 8448 samples: the grid-stride loop goes round for the first 13 warps."""
    _fm_weighted_case(cuda, ROW_WARPS_CAP + 13, 7, E, acc, want, seed=E + 100 * acc + len(want))


def _scale_width(E):
    w = 1
    while w < E and w < 32:
        w <<= 1
    return w


def _field_scale_batch(F, E):
    """A batch past the grid cap (1056 CTAs of 256 / width groups) whose B * F rows are not a multiple of the
    32 / width groups of a warp, so the last warp runs idle groups through the shuffle."""
    w = _scale_width(E)
    B = NUM_SMS * 8 * (256 // w) // F + 1
    while (32 // w) > 1 and (B * F) % (32 // w) == 0:
        B += 1
    return B


def _field_scale_case(cuda, B, F, E, acc, want, seed):
    L, K = _lib(), _kern()
    gen = torch.Generator().manual_seed(seed)
    x, dy = _ints(gen, (B, F * E), -3, 3), _ints(gen, (B, F * E), -3, 3)
    m = _ints(gen, (B, F), -2, 2)
    xw, mw, gw = _put(B, F * E + 3, 1, x, cuda), _put(B, F + 2, 2, m, cuda), _put(B, F * E + 6, 5, dy, cuda)
    y = Window(B, F * E + 4, 3, 1, F * E, F * E, cuda)
    frozen = Frozen(xw.buf, mw.buf, gw.buf)
    xp, mp = xw.buf[:, 1:].data_ptr(), mw.buf[:, 2:].data_ptr()
    _check(L.b2ctr_field_scale_fwd(xp, xw.ld, mp, mw.ld, F, E, y.buf[:, 3:].data_ptr(), y.ld, B, K.stream()),
           "field_scale_fwd")
    y.check_outside("field_scale_fwd")
    dx = Window(B, F * E + 2, 1, 1, F * E, F * E, cuda)
    if acc:
        dx.fill(_ints(gen, (B, 1, F * E), -3, 3).to(cuda))
    dx0 = dx.values().clone()
    dm = Window(B, F + 5, 4, 1, F, F, cuda)
    _check(L.b2ctr_field_scale_bwd(gw.buf[:, 5:].data_ptr(), gw.ld, xp, xw.ld, mp, mw.ld, F, E,
                                   dx.buf[:, 1:].data_ptr() if want != "dm" else None, dx.ld, int(acc),
                                   dm.buf[:, 4:].data_ptr() if want != "dx" else None, dm.ld, B, K.stream()),
           "field_scale_bwd")
    frozen.check("field_scale")
    dx.check_outside("field_scale_bwd dx")
    dm.check_outside("field_scale_bwd dm")
    x64, m64, g64 = (t.to(cuda).double() for t in (x, m, dy))
    x64, g64 = x64.reshape(B, F, E), g64.reshape(B, F, E)
    _same(y.values().reshape(B, F, E), x64 * m64[..., None], "field_scale y")
    if want != "dm":
        _same(dx.values().reshape(B, F, E), g64 * m64[..., None] + (dx0.double().reshape(B, F, E) if acc else 0),
              "field_scale dx")
    else:
        assert torch.equal(dx.values().view(torch.int32), dx0.view(torch.int32)), "field_scale_bwd wrote dx"
    if want != "dx":
        _same(dm.values().reshape(B, F), (g64 * x64).sum(2), "field_scale dm")
    else:
        assert bool((dm.values().view(torch.int32) == NAN_BITS).all()), "field_scale_bwd wrote dm"


@pytest.mark.parametrize("want", WANTS)
@pytest.mark.parametrize("acc", [False, True], ids=["write", "accumulate"])
@pytest.mark.parametrize("E", [1, 2, 3, 5, 9, 17, 33])
def test_field_scale_exact_every_group_width(cuda, E, acc, want):
    """Group widths 1 / 2 / 4 / 8 / 16 / 32 / 32 (two strides), F = 3, a batch past the grid cap with idle groups
    in the last warp."""
    F = 3
    _field_scale_case(cuda, _field_scale_batch(F, E), F, E, acc, want, seed=E + 100 * acc + len(want))


def _softmax_rows_case(cuda, rows, cols, scale, seed):
    """Rows of 1, 2 or 4 maxima (as many as the columns allow) at a random offset in 1/8 steps, the other entries
    128 * k below; dy integers."""
    L, K = _lib(), _kern()
    gen = torch.Generator().manual_seed(seed)
    x = _ints(gen, (rows, cols), -4, -1) * GAP
    nwin = torch.tensor([1, 2, 4])[torch.arange(rows) % 3]
    nwin = torch.minimum(nwin, torch.tensor(1 << (cols.bit_length() - 1)))
    first = torch.argsort(torch.rand((rows, cols), generator=gen), dim=1)
    x[torch.arange(cols)[None, :] < nwin[:, None]] = 0.0                 # placed on the leading columns ...
    x = torch.gather(x, 1, torch.argsort(first, dim=1))                  # ... then scattered by a permutation
    x += _ints(gen, (rows, 1), -40, 40) * 0.125
    dy = _ints(gen, (rows, cols), -3, 3)
    xw, gw = _put(rows, cols + 4, 2, x, cuda), _put(rows, cols + 3, 1, dy, cuda)
    y = Window(rows, cols + 5, 3, 1, cols, cols, cuda)
    frozen = Frozen(xw.buf, gw.buf)
    _check(L.b2ctr_softmax_rows_fwd(xw.buf[:, 2:].data_ptr(), xw.ld, y.buf[:, 3:].data_ptr(), y.ld, rows, cols, scale,
                                    K.stream()), "softmax_rows_fwd")
    y.check_outside("softmax_rows_fwd")
    frozen_y = Frozen(y.buf)
    dx = Window(rows, cols + 2, 1, 1, cols, cols, cuda)
    _check(L.b2ctr_softmax_rows_bwd(y.buf[:, 3:].data_ptr(), y.ld, gw.buf[:, 1:].data_ptr(), gw.ld,
                                    dx.buf[:, 1:].data_ptr(), dx.ld, rows, cols, scale, K.stream()), "softmax_rows_bwd")
    frozen.check("softmax_rows")
    frozen_y.check("softmax_rows_bwd")
    dx.check_outside("softmax_rows_bwd")
    p, n, _ = _exact_softmax(x.to(cuda).double(), "softmax_rows")
    want_y = scale * p
    g64 = dy.to(cuda).double()
    # y = scale / n on the maxima: (13/2) * 2^-k for scale 26; dx = y (dy - <y, dy> / scale) = y (dy - <p, dy>)
    _fits(want_y * (g64.abs() + (p * g64.abs()).sum(1, keepdim=True)), scale / 4 / 4 / 4, "softmax_rows dx")
    _same(y.values().reshape(rows, cols), want_y, "softmax_rows y")
    _same(dx.values().reshape(rows, cols), want_y * (g64 - (p * g64).sum(1, keepdim=True)), "softmax_rows dx")
    assert bool((n <= 4).all())


@pytest.mark.parametrize("scale", [1.0, 26.0])
@pytest.mark.parametrize("cols", [1, 31, 32, 33, 64, 100])
def test_softmax_rows_exact_past_the_grid_cap(cuda, cols, scale):
    _softmax_rows_case(cuda, ROW_WARPS_CAP + 37, cols, scale, seed=cols + int(scale))


@pytest.mark.parametrize("E", [1, 31, 33, 65])
def test_fm_weighted_random_data_within_tolerance(cuda, E):
    _check_fm(cuda, ROW_WARPS_CAP + 13, 7, E, E)


@pytest.mark.parametrize("E", [2, 3, 9, 17, 33])
def test_field_scale_random_data_within_tolerance(cuda, E):
    _check_scale(cuda, 1001, 3, E, E)


@pytest.mark.parametrize("cols", [31, 33, 100])
def test_softmax_rows_random_data_within_tolerance(cuda, cols):
    """IFM's scale F = 26 on normal logits (with one large one: the maximum is subtracted first)."""
    K = _kern()
    gen = torch.Generator().manual_seed(cols)
    rows = ROW_WARPS_CAP + 37
    xb = (torch.randn((rows, cols + 5), generator=gen) * 3).to(cuda)
    xb[:, 2] += 60.0
    x = xb[:, 2:2 + cols]
    y = K.softmax_rows_fwd(x, 26.0)
    x64 = x.double().requires_grad_(True)
    ref = 26.0 * torch.softmax(x64, dim=1)
    _close(y, ref, "softmax y", 1e-6)
    g = torch.randn((rows, cols), generator=gen).to(cuda)
    dx = K.softmax_rows_bwd(y, g, 26.0)
    (ref * g.double()).sum().backward()
    err = float((dx.double() - x64.grad).abs().max())
    assert err <= 1e-5 * float((ref.detach().abs() * g.double().abs()).max()) + 1e-30, "softmax dx: %g" % err
