"""GPU: the DIN, sequence-pooling, BatchNormalization / Dice, dropout, LayerNorm and ONN field-aware kernels exactly,
at their block, grid and template boundaries, with NaN in every padding.

The operands are small integers (times a power of two), and every check first asserts, from the data, that the sum
of the absolute values of the terms of each result stays below 2^24 units of its grid, so every partial sum in every
order is exact in fp32.  Where a kernel rounds once by an IEEE operation (division, sqrtf, __f*_rn, a lone product)
the reference restates that rounding in fp32 from exact intermediates.  Softmaxes are made exact as in
test_attention_kernels_exact_gpu: every valid score is its row's maximum or at least 128 below it, with a
power-of-two count of maxima; a row with no valid position gets 1/T, one fp32 rounding.  BatchNormalization / Dice
get var = 4^-j with eps = 0, so rsqrtf gives 2^j (a one-row probe asserts that the device's rsqrtf is exact
there), and Dice's x are either the mean or at least 128 / rs from it, so p is 1/2, 0 or 1 exactly.  Inputs are
windows of NaN-filled buffers (pitch gaps and rows past the batch hold a NaN with a payload); outputs, saved state
and workspaces are NaN-filled, and nothing outside them may change, bit for bit.

* b2ctr_dropout against a numpy uint64 restatement of mix32 and of thr = (uint32_t)(rate * 2^32), keep_scale in
  fp32; rate 0 / 0.25 / 0.5 / 0.9, seeds next to 2^64, n around the grid cap; and the mask the exact MHA test takes
  from b2ctr_dropout is the restated one;
* b2ctr_seqpool_fwd / _bwd (sum / mean / max) with masks that are not prefixes (bytes 1, 2 and 255) and with
  lengths, empty bags, ties, B*E across the 270,336-thread cap; b2ctr_seqweight (plain and soft-maxed) across its
  135,168-sample cap; b2ctr_seqscale across the 270,336-thread cap;
* b2ctr_din_att_input_fwd / _bwd on q / keys windows, T 1 / 7 / 50 / 200 x E 1 / 8 / 64 / 100, B*E around the
  backward's 270,336-thread cap, and the C4 shape B = 8192, T = 50, E = 64;
* b2ctr_din_pool_fwd / _bwd in all four (weight_norm, return_score) modes, T on both sides of 32 and 64, B around
  one CTA and the 8,448-warp grid cap, rows with every position masked;
* b2ctr_colstats, b2ctr_bn_apply, b2ctr_bn_bwd, b2ctr_dice_fwd, b2ctr_dice_bwd at m 1 / 511 / 512 / 513 / 1024
  against every n in 1 / 40 / 80 / 128 / 129 / 255 / 256 / 257 / 1300, at m = 409,600 (DIN's B*T at C4) and
  409,601, and at ONN's BatchNormalization shape 65,536 x 1300, with NaN workspaces.  Column statistics, sums,
  dgamma / dbeta, dalpha, every forward, inference dx and Dice's training dx are bit-exact at every m;
  BatchNormalization's training dx is bit-exact when m is a power of two and within 6 ulp of its terms otherwise
  (its xn * sum(dy xn) / m term rounds in an order the compiler may contract);
* b2ctr_layernorm_fwd / _bwd at n 1 .. 1024 (every NK instantiation and idle lanes) x rows 1 / 7 / 8 / 9 and around
  the backward's 2,112-row pass, and at BST's 409,600 and 409,601 rows, with and without the residual and
  gamma / beta / dgamma / dbeta; every partial row of the NaN workspace is written.  dx is bit-exact for n a power of
  two and otherwise equals the fp32 restatement, with or without the fma contraction of each of its two products;
* b2ctr_ffm_product_fwd / _bwd (both modes) at F 2 / 3 / 32 / 33 / 64 x E 1 / 3 / 4 / 5 / 64, the float4 and
  scalar paths, B around one CTA and the 8,448-warp grid cap and 65,537; int32 / int64 / strided ids, hashed fields
  (oracle/farmhash.py), pooled fields, out-of-range ids (zero rows, counted once, gradient rows still written), every
  gradient slot written once; ONN's bench shape (26 x 1M, E = 4, B = 65,536); FieldAwarePlan refuses tables that
  are not 16-byte aligned before it launches anything;
* random data within the tolerances of test_simt_kernels_gpu / test_bst_gpu at the C4, BST and ONN shapes.
"""
import numpy as np
import pytest
import torch

import test_bst_gpu as BST
import test_simt_kernels_gpu as SIMT
from test_attention_kernels_exact_gpu import (GAP, MHA_B, MHA_D, MHA_HEADS, MHA_RUNS, MHA_T, NUM_SMS, PAD_SCORE, _check,
                                              _exact_softmax, _ints, _kern, _nan_workspace, _pow2, _put, _round32)
from test_attention_kernels_exact_gpu import Flat as _Flat
from test_product_kernels_exact_gpu import NAN_BITS, Frozen, Window, _fits, _lib, _same

pytestmark = pytest.mark.gpu

THREAD_CAP = NUM_SMS * 8 * 256           # grid_for(n, 256, 8): 1056 CTAs of 256 threads = 270,336
WARP_CAP = NUM_SMS * 8 * 8               # grid_for(B, 8, 8): 1056 CTAs of 8 warps = 8,448 rows
SEQW_CAP = NUM_SMS * 8 * 128             # seqweight: grid_for(B, 128, 8) = 135,168 samples
STAT_ROWS = 512                          # kStatRows: rows per block of the column reductions
LN_PASS = 2 * NUM_SMS * 8                # layernorm_bwd: 264 CTAs of 8 warps = 2,112 rows per pass
M64 = (1 << 64) - 1


class Flat(_Flat):
    """A Flat whose NaN tail (at least 9 floats) pads the buffer to a multiple of 1024 floats, so that ``_freeze``
    digests it by rows of 1024 rather than one chunk per 1024 floats."""

    def __init__(self, n, device):
        super().__init__(n, device, tail=9 + (-(n + 9)) % 1024)


def _freeze(*bufs):
    return Frozen(*[b.view(-1, 1024) if b.dim() == 1 and b.numel() % 1024 == 0 else b for b in bufs])


def _flat(vals, device):
    """A Flat (NaN tail) holding ``vals``."""
    f = Flat(vals.numel(), device)
    f.values()[:] = vals.reshape(-1).to(device)
    return f


def _dev_ints(gen, shape, lo, hi):
    """Integers in [lo, hi] as fp32, drawn on the generator's device (the large operands)."""
    return torch.randint(lo, hi + 1, tuple(shape), generator=gen, device=gen.device).to(torch.float32)


def _bytes(vals, device):
    """uint8 ``vals`` at the front of a buffer whose tail holds 0x5a (a multiple of 4096 bytes long)."""
    n = vals.numel()
    buf = torch.full(((n + 16 + 4095) // 4096 * 4096,), 0x5a, dtype=torch.uint8, device=device)
    buf[:n] = vals.reshape(-1).to(device)
    return buf


def _masks(gen, B, T, p=0.6):
    """uint8 validity masks that are not prefixes: valid bytes are 1, 2 or 255; row 0 is empty, row 1 full."""
    m = torch.tensor([1, 2, 255], dtype=torch.uint8)[torch.randint(0, 3, (B, T), generator=gen)]
    m[torch.rand((B, T), generator=gen) >= p] = 0
    m[0] = 0
    if B > 1:
        m[1] = torch.tensor([255, 2, 1], dtype=torch.uint8)[torch.arange(T) % 3]
    return m


def _lengths(gen, B, T):
    ln = torch.randint(0, T + 1, (B,), generator=gen, dtype=torch.int32)
    ln[0] = 0
    if B > 1:
        ln[1] = T
    return ln, torch.arange(T)[None, :] < ln[:, None].long()


def _gapped_scores(gen, valid):
    """Scores whose softmax over the valid positions is exact: 1, 2 or 4 maxima (as many as the row's valid count
    allows) at a row offset in 1/8 steps, every other valid score 128 k (k = 1..4) below; NaN where invalid."""
    B, T = valid.shape
    nv = valid.sum(1)
    cap = torch.where(nv >= 4, 4, torch.where(nv >= 2, 2, 1))
    nw = torch.minimum(torch.tensor([1, 2, 4])[torch.randint(0, 3, (B,), generator=gen)], cap)
    key = torch.rand((B, T), generator=gen)
    key[~valid] = 2.0
    rank = torch.argsort(torch.argsort(key, 1), 1)
    win = (rank < nw[:, None]) & valid
    off = _ints(gen, (B, 1), -40, 40) * 0.125
    s = torch.where(win, off.expand(B, T), off - GAP * _ints(gen, (B, T), 1, 4))
    s[~valid] = float("nan")
    return s


def _softmax_weights(score, valid):
    """float64 weights of the masked softmax: 1/n on the n maxima; 1/T rounded once to fp32 on a row with no
    valid position (T equal paddings)."""
    S = torch.where(valid, score.double(), torch.full((), PAD_SCORE, dtype=torch.float64, device=score.device))
    p, n, _ = _exact_softmax(S, "masked scores", valid)
    return torch.where(_pow2(n), p, _round32(p))


# ================================================================================================ dropout
GOLDEN = 0x9E3779B97F4A7C15


def _mix32(z):
    """common.cuh's mix32 on uint64 numpy arrays (multiplication wraps mod 2^64)."""
    with np.errstate(over="ignore"):
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xbf58476d1ce4e5b9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94d049bb133111eb)
        return ((z ^ (z >> np.uint64(31))) >> np.uint64(32)).astype(np.uint32)


def _dropout_keep(n, rate, seed):
    """Element i survives iff mix32(seed * 0x9E3779B97F4A7C15 + i) >= (uint32_t)(rate * 2^32), rate an fp32
    promoted to double; -> (bool [n], fp32 keep scale 1 / (1 - rate))."""
    with np.errstate(over="ignore"):
        z = np.uint64((seed * GOLDEN) & M64) + np.arange(n, dtype=np.uint64)
    thr = int(float(np.float32(rate)) * 4294967296.0)
    scale = np.float32(1.0) / (np.float32(1.0) - np.float32(rate))
    return torch.from_numpy(_mix32(z) >= np.uint32(thr)), float(scale)


DROP_N = [1, 255, THREAD_CAP - 1, THREAD_CAP, THREAD_CAP + 1, 2 * THREAD_CAP + 1]
DROP_SEEDS = [0, 1, 0x1234567, M64 - 1, M64]


@pytest.mark.parametrize("rate", [0.0, 0.25, 0.5, 0.9])
@pytest.mark.parametrize("n", DROP_N, ids=["one", "cta_minus_1", "cap_minus_1", "cap", "cap_plus_1", "two_caps_plus_1"])
def test_dropout_matches_the_restated_hash(cuda, n, rate):
    assert THREAD_CAP == 270336 and -(-(THREAD_CAP + 1) // 256) > NUM_SMS * 8
    K = _kern()
    gen = torch.Generator().manual_seed(n)
    x = _flat(_ints(gen, (n,), -7, 7) * 0.25, cuda)
    frozen = _freeze(x.buf)
    for seed in DROP_SEEDS:
        keep, scale = _dropout_keep(n, rate, seed)
        y = Flat(n, cuda)
        _check(_lib().b2ctr_dropout(x.buf.data_ptr(), y.buf.data_ptr(), n, rate, seed, K.stream()), "dropout")
        frozen.check("dropout")
        y.check_outside("dropout")
        want = torch.where(keep.to(cuda), _round32(x.values().double() * scale), torch.zeros((), dtype=torch.float64,
                                                                                           device=cuda))
        _same(y.values(), want, "dropout rate %g seed %#x" % (rate, seed))
        if rate == 0.0:
            assert bool(keep.all())


def test_mha_dropout_mask_is_the_restated_hash(cuda):
    """The exact MHA test takes its dropout mask from b2ctr_dropout on ones (the attention kernels share mix32):
    at every shape and seed it uses, that mask is the restated one, keep scale 2."""
    K = _kern()
    for d in MHA_D:
        for T in MHA_T:
            for run, (_, _, rate, _) in MHA_RUNS.items():
                if not rate:
                    continue
                seed = 1000 * d + T + len(run)
                n = MHA_HEADS * MHA_B * T * T
                got = K.dropout(torch.ones(n, device=cuda), rate, seed)
                keep, scale = _dropout_keep(n, rate, seed)
                assert scale == 2.0
                _same(got, keep.to(cuda).double() * 2.0, "mha dropout mask d=%d T=%d" % (d, T))


# ================================================================================================ sequence pooling
def _seqpool_case(cuda, B, T, E, kind, seed):
    L, K = _lib(), _kern()
    gen = torch.Generator().manual_seed(seed)
    x = _ints(gen, (B, T, E), -2, 2)                  # |x| <= 2: every masked x - 1e9 rounds to -1e9 and ties
    dout = _ints(gen, (B, E), -12, 12)
    if kind == "mask":
        mask = _masks(gen, B, T)
        valid, mk, ln = mask != 0, _bytes(mask, cuda), None
    else:
        lens, valid = _lengths(gen, B, T)
        mk, ln = None, lens.to(cuda)
    xf, gf = _flat(x, cuda), _flat(dout, cuda)
    frozen = _freeze(*[t for t in (xf.buf, gf.buf, mk, ln) if t is not None])
    x64, g64, v = x.to(cuda).double(), dout.to(cuda).double(), valid.to(cuda)[..., None]
    Lf = _round32(v.sum(1).double() + float(np.float32(1e-8)))          # L + 1e-8f in fp32
    masked = torch.where(v, x64, _round32(x64 - 1e9))
    mx = masked.max(1).values
    cnt = (masked == mx[:, None]).sum(1).double()
    _fits((x64.abs() * v).sum(1), 1.0, "seqpool sum")
    zero = torch.zeros((), dtype=torch.float64, device=cuda)
    for mode, name in ((1, "sum"), (2, "mean"), (3, "max")):
        out, dx = Flat(B * E, cuda), Flat(B * T * E, cuda)
        p = lambda t: t.data_ptr() if t is not None else None          # noqa: E731
        _check(L.b2ctr_seqpool_fwd(xf.buf.data_ptr(), p(mk), p(ln), out.buf.data_ptr(), B, T, E, mode, K.stream()),
               "seqpool_fwd")
        _check(L.b2ctr_seqpool_bwd(xf.buf.data_ptr(), p(mk), p(ln), gf.buf.data_ptr(), dx.buf.data_ptr(), B, T, E,
                                   mode, K.stream()), "seqpool_bwd")
        frozen.check("seqpool " + name)
        out.check_outside("seqpool_fwd " + name)
        dx.check_outside("seqpool_bwd " + name)
        S = (x64 * v).sum(1)
        if mode == 1:
            want, wdx = S, torch.where(v, g64[:, None], zero)
        elif mode == 2:
            want, wdx = _round32(S / Lf), torch.where(v, _round32(g64 / Lf)[:, None], zero)
        else:
            want, wdx = mx, torch.where(masked == mx[:, None], _round32(g64 / cnt)[:, None], zero)
        _same(out.values().reshape(B, E), want, "seqpool_fwd %s (%s)" % (name, kind))
        _same(dx.values().reshape(B, T, E), wdx, "seqpool_bwd %s (%s)" % (name, kind))


@pytest.mark.parametrize("kind", ["mask", "len"])
@pytest.mark.parametrize("E", [1, 8, 33])
@pytest.mark.parametrize("T", [1, 7, 50])
def test_seqpool_exact(cuda, T, E, kind):
    _seqpool_case(cuda, 37, T, E, kind, seed=100 * T + E + len(kind))


SEQ_CAP_B = [THREAD_CAP // 8 - 1, THREAD_CAP // 8, THREAD_CAP // 8 + 1, 2 * THREAD_CAP // 8 + 1]


@pytest.mark.parametrize("kind", ["mask", "len"])
@pytest.mark.parametrize("B", SEQ_CAP_B, ids=["cap_minus_1", "cap", "cap_plus_1", "two_caps_plus_1"])
def test_seqpool_exact_across_the_grid_cap(cuda, B, kind):
    """E = 8: one thread per (b, e), B * E around the 270,336 threads of a full grid."""
    assert (THREAD_CAP // 8) * 8 == THREAD_CAP
    _seqpool_case(cuda, B, 7, 8, kind, seed=B + len(kind))


def test_seqpool_mean_divides_by_the_valid_positions(cuda):
    """Mask bytes 2 and 255 are one valid position each: the mean divides by the count of non-zero bytes."""
    L, K = _lib(), _kern()
    B, T, E = 4, 6, 3
    mask = torch.tensor([[2, 0, 2, 0, 0, 0], [255, 255, 0, 1, 0, 0], [0, 0, 0, 0, 0, 255], [2, 255, 1, 2, 255, 1]],
                        dtype=torch.uint8)
    x = torch.arange(B * T * E, dtype=torch.float32).reshape(B, T, E)
    xf, mk = _flat(x, cuda), _bytes(mask, cuda)
    out = Flat(B * E, cuda)
    _check(L.b2ctr_seqpool_fwd(xf.buf.data_ptr(), mk.data_ptr(), None, out.buf.data_ptr(), B, T, E, 2, K.stream()),
           "seqpool_fwd")
    v = (mask != 0)[..., None].double()
    want = _round32((x.double() * v).sum(1) / v.sum(1))
    _same(out.values().reshape(B, E).cpu(), want, "seqpool mean with mask bytes 2 / 255")
    dx = Flat(B * T * E, cuda)
    g = _flat(torch.full((B, E), 6.0), cuda)
    _check(L.b2ctr_seqpool_bwd(xf.buf.data_ptr(), mk.data_ptr(), None, g.buf.data_ptr(), dx.buf.data_ptr(), B, T, E,
                               2, K.stream()), "seqpool_bwd")
    _same(dx.values().reshape(B, T, E).cpu(), (_round32(6.0 / v.sum(1, keepdim=True)) * v).expand(B, T, E),
          "seqpool mean backward")


def _seqweight_case(cuda, B, T, kind, norm, seed):
    L, K = _lib(), _kern()
    gen = torch.Generator().manual_seed(seed)
    if kind == "mask":
        mask = _masks(gen, B, T)
        valid, mk, ln = mask != 0, _bytes(mask, cuda), None
    else:
        lens, valid = _lengths(gen, B, T)
        mk, ln = None, lens.to(cuda)
    w = _gapped_scores(gen, valid)
    wf = _flat(w, cuda)
    wt = Flat(B * T, cuda)
    frozen = _freeze(*[t for t in (wf.buf, mk, ln) if t is not None])
    _check(L.b2ctr_seqweight(wf.buf.data_ptr(), mk.data_ptr() if mk is not None else None,
                             ln.data_ptr() if ln is not None else None, wt.buf.data_ptr(), B, T, int(norm),
                             K.stream()), "seqweight")
    frozen.check("seqweight")
    wt.check_outside("seqweight")
    vd = valid.to(cuda)
    if norm:
        want = _softmax_weights(wf.values().reshape(B, T), vd)
    else:
        want = torch.where(vd, wf.values().reshape(B, T).double(), torch.zeros((), dtype=torch.float64, device=cuda))
    _same(wt.values().reshape(B, T), want, "seqweight norm=%d (%s)" % (norm, kind))
    return wt.values().reshape(B, T)


@pytest.mark.parametrize("norm", [0, 1])
@pytest.mark.parametrize("kind", ["mask", "len"])
@pytest.mark.parametrize("B", [1, 37, SEQW_CAP - 1, SEQW_CAP, SEQW_CAP + 1],
                         ids=["one", "b37", "cap_minus_1", "cap", "cap_plus_1"])
def test_seqweight_exact_across_the_grid_cap(cuda, B, kind, norm):
    """One thread per sample, B around 1056 CTAs x 128 threads; T = 5 (1/5 rounds) on masks, 8 on lengths."""
    assert SEQW_CAP == 135168
    _seqweight_case(cuda, B, 5 if kind == "mask" else 8, kind, norm, seed=B + norm)


@pytest.mark.parametrize("rows", [THREAD_CAP // 8 - 1, THREAD_CAP // 8, THREAD_CAP // 8 + 1],
                         ids=["cap_minus_1", "cap", "cap_plus_1"])
def test_seqscale_exact_across_the_grid_cap(cuda, rows):
    """out = x * wt[row] rounded once, with the soft-maxed weights (1/n, 0 and fp32 1/5) of seqweight; E = 8."""
    L, K = _lib(), _kern()
    E, T = 8, 5
    assert rows * E - THREAD_CAP in (-8, 0, 8)
    wt = _seqweight_case(cuda, -(-rows // T), T, "mask", 1, seed=rows).reshape(-1)[:rows].contiguous()
    x = _flat(_ints(torch.Generator().manual_seed(rows), (rows, E), -7, 7), cuda)
    wf = _flat(wt, cuda)
    out = Flat(rows * E, cuda)
    frozen = _freeze(x.buf, wf.buf)
    _check(L.b2ctr_seqscale(x.buf.data_ptr(), wf.buf.data_ptr(), out.buf.data_ptr(), rows, E, K.stream()), "seqscale")
    frozen.check("seqscale")
    out.check_outside("seqscale")
    _same(out.values().reshape(rows, E), _round32(x.values().reshape(rows, E).double() * wt.double()[:, None]),
          "seqscale")


# ================================================================================================ DIN
def _din_input_case(cuda, B, T, E, seed):
    L, K = _lib(), _kern()
    gen = torch.Generator(device=cuda).manual_seed(seed)
    q, k = _dev_ints(gen, (B, E), -3, 3), _dev_ints(gen, (B, T * E), -3, 3)
    qw, kw = _put(B, E + 5, 2, q, cuda), _put(B, T * E + 7, 3, k, cuda)
    qp, kp = qw.buf[:, 2:].data_ptr(), kw.buf[:, 3:].data_ptr()
    out = Flat(B * T * 4 * E, cuda)
    frozen = _freeze(qw.buf, kw.buf)
    _check(L.b2ctr_din_att_input_fwd(qp, qw.ld, kp, kw.ld, out.buf.data_ptr(), B, T, E, K.stream()),
           "din_att_input_fwd")
    out.check_outside("din_att_input_fwd")
    g = _flat(_dev_ints(gen, (B * T * 4 * E,), -3, 3), cuda)
    dq, dk = Flat(B * E, cuda), Flat(B * T * E, cuda)
    frozen_g = _freeze(g.buf, out.buf)
    _check(L.b2ctr_din_att_input_bwd(qp, qw.ld, kp, kw.ld, g.buf.data_ptr(), dq.buf.data_ptr(), dk.buf.data_ptr(), B,
                                     T, E, K.stream()), "din_att_input_bwd")
    frozen.check("din_att_input")
    frozen_g.check("din_att_input_bwd")
    dq.check_outside("din_att_input_bwd dq")
    dk.check_outside("din_att_input_bwd dk")
    chunk = max(1, (1 << 24) // (T * E))
    for b0 in range(0, B, chunk):
        sl = slice(b0, min(B, b0 + chunk))
        n = sl.stop - b0
        q64 = q[sl].to(cuda).double()[:, None, :].expand(n, T, E)
        k64 = k[sl].to(cuda).double().reshape(n, T, E)
        o = out.values().reshape(B, T, 4, E)[sl]
        for i, want in enumerate((q64, k64, q64 - k64, q64 * k64)):
            _same(o[:, :, i], want, "din_att_input_fwd block %d" % i)
        g64 = g.values().reshape(B, T, 4, E)[sl].double()
        _fits((g64[:, :, 0].abs() + g64[:, :, 2].abs() + (g64[:, :, 3] * k64).abs()).sum(1), 1.0, "din dq")
        _same(dq.values().reshape(B, E)[sl], (g64[:, :, 0] + g64[:, :, 2] + g64[:, :, 3] * k64).sum(1), "din dq")
        _same(dk.values().reshape(B, T, E)[sl], g64[:, :, 1] - g64[:, :, 2] + g64[:, :, 3] * q64, "din dkeys")


@pytest.mark.parametrize("E", [1, 8, 64, 100])
@pytest.mark.parametrize("T", [1, 7, 50, 200])
def test_din_attention_input_exact(cuda, T, E):
    _din_input_case(cuda, 37, T, E, seed=1000 * T + E)


@pytest.mark.parametrize("B", [THREAD_CAP // 64 - 1, THREAD_CAP // 64, THREAD_CAP // 64 + 1, 8192],
                         ids=["cap_minus_1", "cap", "cap_plus_1", "c4"])
def test_din_attention_input_exact_across_the_backward_cap(cuda, B):
    """E = 64: the backward's one thread per (b, e) at B * E around 270,336; B = 8192 with T = 50 is C4's shape."""
    assert (THREAD_CAP // 64) * 64 == THREAD_CAP
    _din_input_case(cuda, B, 50 if B == 8192 else 7, 64, seed=B)


def _din_pool_case(cuda, B, T, E, seed):
    L, K = _lib(), _kern()
    gen = torch.Generator().manual_seed(seed)
    mask = _masks(gen, B, T)
    mask[4::5] = 0                                     # every fifth row: every position masked
    valid = mask != 0
    score = _gapped_scores(gen, valid)
    keys = _ints(gen, (B, T, E), -2, 2)                # 0, +-1, +-2: a product with 1/T is exact
    empty = ~valid.any(1)
    one = torch.arange(T)[None, :] == (torch.arange(B) % T)[:, None]
    keys[empty[:, None] & ~one] = 0                    # a row that sees no position keeps one key row
    sf, mk = _flat(score, cuda), _bytes(mask, cuda)
    kw = _put(B, T * E + 5, 1, keys.reshape(B, T * E), cuda)
    kp = kw.buf[:, 1:].data_ptr()
    vd, k64 = valid.to(cuda), keys.to(cuda).double()
    zero = torch.zeros((), dtype=torch.float64, device=cuda)
    for wn in (0, 1):
        for rs in (0, 1):
            what = "din_pool weight_norm=%d return_score=%d" % (wn, rs)
            w, out = Flat(B * T, cuda), Flat(B * (T if rs else E), cuda)
            frozen = _freeze(sf.buf, mk, kw.buf)
            _check(L.b2ctr_din_pool_fwd(sf.buf.data_ptr(), kp, kw.ld, mk.data_ptr(), w.buf.data_ptr(),
                                        out.buf.data_ptr(), B, T, E, wn, rs, K.stream()), "din_pool_fwd")
            w.check_outside(what + " w")
            out.check_outside(what + " out")
            ww = _softmax_weights(sf.values().reshape(B, T), vd) if wn else \
                torch.where(vd, sf.values().reshape(B, T).double(), zero)
            _same(w.values().reshape(B, T), ww, what + " weights")
            if rs:
                _same(out.values().reshape(B, T), ww, what + " out")
            else:
                _fits((ww.abs()[..., None] * k64.abs()).sum(1)[~empty.to(cuda)], 2.0 ** -5, what + " out")
                _same(out.values().reshape(B, E), (ww[..., None] * k64).sum(1), what + " out")
            dout = _flat(_ints(gen, (B, T if rs else E), -3, 3), cuda)
            ds, dk = Flat(B * T, cuda), Flat(B * T * E, cuda)
            frozen_b = _freeze(dout.buf, w.buf)
            _check(L.b2ctr_din_pool_bwd(w.buf.data_ptr(), kp, kw.ld, mk.data_ptr(), dout.buf.data_ptr(),
                                        ds.buf.data_ptr(), dk.buf.data_ptr(), B, T, E, wn, rs, K.stream()),
                   "din_pool_bwd")
            frozen.check(what)
            frozen_b.check(what + " bwd")
            ds.check_outside(what + " dscore")
            dk.check_outside(what + " dkeys")
            g64 = dout.values().reshape(B, -1).double()
            dsw = g64 if rs else (g64[:, None, :] * k64).sum(2)
            if wn:
                dsw = torch.where(vd, ww * (dsw - (ww * dsw).sum(1, keepdim=True)), zero)
            else:
                dsw = torch.where(vd, dsw, zero)
            _same(ds.values().reshape(B, T), dsw, what + " dscore")
            if rs:
                assert bool((dk.buf.view(torch.int32) == NAN_BITS).all()), what + ": dkeys written"
            else:
                _same(dk.values().reshape(B, T, E), _round32(ww[..., None] * g64[:, None, :]), what + " dkeys")


DIN_POOL_T = [1, 31, 32, 33, 64, 65]
DIN_POOL_B = [1, 8, WARP_CAP - 1, WARP_CAP, WARP_CAP + 1, 2 * WARP_CAP + 1]


@pytest.mark.parametrize("B", DIN_POOL_B, ids=["one", "cta", "cap_minus_1", "cap", "cap_plus_1", "two_caps_plus_1"])
@pytest.mark.parametrize("T", DIN_POOL_T)
def test_din_pool_exact(cuda, T, B):
    """One warp per sample: T on both sides of one and two lane rounds; B around one CTA and 1056 x 8 warps."""
    assert WARP_CAP == 8448
    _din_pool_case(cuda, B, T, 3, seed=100 * T + B)


@pytest.mark.parametrize("E", [1, 33, 64, 100])
def test_din_pool_exact_wide_keys(cuda, E):
    _din_pool_case(cuda, 37, 50, E, seed=E)


# ================================================================================================ BatchNorm / Dice
BN_M = [1, 511, 512, 513, 1024]
BN_N = [1, 40, 80, 128, 129, 255, 256, 257, 1300]
BN_BIG = [(409600, 40), (409600, 129), (409601, 1), (409601, 257), (65536, 1300)]


def _rsqrt_probe(cuda, js):
    """bn_apply on one row with x - mean = 1, var = 4^-j, eps = 0: y is the device's rsqrtf(4^-j), which the exact
    cases take to be 2^j."""
    K = _kern()
    n = len(js)
    j = torch.tensor(js, dtype=torch.float64)
    y = K.bn_apply(torch.ones((1, n), device=cuda), torch.zeros(n, device=cuda),
                   (4.0 ** -j).float().to(cuda), None, None, 1, n, 0.0)
    assert torch.equal(y[0].double().cpu(), 2.0 ** j), "rsqrtf(4^-j) is not 2^j on this device: %s" % y


BN_J, DICE_J = [1, 2, 3], [5, 6]


def _col(gen, n, vals):
    return torch.tensor(vals, dtype=torch.float32, device=gen.device)[
        torch.randint(0, len(vals), (n,), generator=gen, device=gen.device)]


def _bn_dice_operands(gen, m, n):
    """Column means mu odd in [-3, 3].  BatchNorm: x = mu + d / rs (d in [-2, 2]) so xn = d; dy in [-2, 2];
    gamma +-1/2, +-1, +-2; beta in 1/4.  Dice: x = mu + k * 128 / rs (k in -1..1, zero-sum per column, so the mean
    is mu; 128 / rs is 4 or 2, so every x is odd and a dropped row moves its column's sum); alpha in 1/2 steps."""
    dev = gen.device
    mu = _dev_ints(gen, (n,), -2, 1) * 2 + 1
    rs_bn = 2.0 ** _col(gen, n, BN_J)
    x_bn = mu + _dev_ints(gen, (m, n), -2, 2) / rs_bn
    rs_d = 2.0 ** _col(gen, n, DICE_J)
    h = m // 2
    k = _dev_ints(gen, (h, n), -1, 1)
    kk = torch.cat([k, -k, torch.zeros((m - 2 * h, n), device=dev)])[torch.randperm(m, generator=gen, device=dev)]
    x_d = mu + kk * (GAP / rs_d)
    return dict(mu=mu, var_bn=1.0 / (rs_bn * rs_bn), var_d=1.0 / (rs_d * rs_d), x_bn=x_bn, x_d=x_d,
                dy=_dev_ints(gen, (m, n), -2, 2), gamma=_col(gen, n, [-2.0, -1.0, -0.5, 0.5, 1.0, 2.0]),
                beta=_dev_ints(gen, (n,), -5, 5) * 0.25, alpha=_dev_ints(gen, (n,), -2, 2) * 0.5)


def _bn_dice_case(cuda, m, n, seed):
    L, K = _lib(), _kern()
    gen = torch.Generator(device=cuda).manual_seed(seed)
    _rsqrt_probe(cuda, BN_J + DICE_J)
    o = _bn_dice_operands(gen, m, n)
    st = K.stream()
    d64 = lambda t: t.to(cuda).double()                 # noqa: E731
    zero = torch.zeros((), dtype=torch.float64, device=cuda)
    invm = float(np.float32(1.0) / np.float32(m))
    pow2m = m & (m - 1) == 0

    # ---- colstats over a window (ld = n + 3) of Dice's x; NaN workspace
    xw = _put(m, n + 3, 1, o["x_d"], cuda)
    stats = Flat(2 * n, cuda)
    nb = L.b2ctr_colstats_workspace_bytes(m, n)
    assert nb == (3 * (-(-m // STAT_ROWS)) * n + 3 * n) * 4
    ws = _nan_workspace(nb, cuda)
    frozen = _freeze(xw.buf)
    _check(L.b2ctr_colstats(xw.buf[:, 1:].data_ptr(), xw.ld, m, n, stats.buf.data_ptr(), ws.data_ptr(), nb, st),
           "colstats")
    frozen.check("colstats")
    stats.check_outside("colstats")
    assert bool((ws[nb // 4:].view(torch.int32) == NAN_BITS).all()), "colstats wrote past its workspace"
    x64 = d64(o["x_d"])
    _fits(x64.abs().sum(0), 1.0, "colstats sum")
    mean = _round32(x64.sum(0) * invm)                   # fp32(S) * fp32(1 / m), rounded once
    assert torch.equal(mean, d64(o["mu"])), "the restated mean is not on the operand grid"
    _fits(((x64 - mean) ** 2).sum(0), 1.0, "colstats sum of squares")
    _same(stats.values()[:n], mean, "colstats mean")
    _same(stats.values()[n:], _round32(((x64 - mean) ** 2).sum(0) * invm), "colstats variance")
    del xw, ws

    # ---- BatchNormalization: bn_apply, bn_bwd (inference and training), gamma / beta as tensors and NULL
    xb, dyf = _flat(o["x_bn"], cuda), _flat(o["dy"], cuda)
    meanf, varf = _flat(o["mu"], cuda), _flat(o["var_bn"], cuda)
    gf, bf = _flat(o["gamma"], cuda), _flat(o["beta"], cuda)
    frozen = _freeze(xb.buf, dyf.buf, meanf.buf, varf.buf, gf.buf, bf.buf)
    rs = 1.0 / d64(o["var_bn"]).sqrt()
    xn = (d64(o["x_bn"]) - d64(o["mu"])) * rs
    dy = d64(o["dy"])
    S1, S2 = dy.sum(0), (dy * xn).sum(0)
    _fits(dy.abs().sum(0), 1.0, "bn sum dy")
    _fits((dy * xn).abs().sum(0), 1.0, "bn sum dy xn")
    for affine in (True, False):
        g_, b_ = (gf, bf) if affine else (None, None)
        gm = d64(o["gamma"]) if affine else torch.ones(n, dtype=torch.float64, device=cuda)
        p = lambda f: f.buf.data_ptr() if f is not None else None     # noqa: E731
        y = Flat(m * n, cuda)
        _check(L.b2ctr_bn_apply(xb.buf.data_ptr(), meanf.buf.data_ptr(), varf.buf.data_ptr(), p(g_), p(b_),
                                y.buf.data_ptr(), m, n, 0.0, st), "bn_apply")
        y.check_outside("bn_apply")
        _same(y.values().reshape(m, n), xn * gm + (d64(o["beta"]) if affine else 0), "bn_apply affine=%s" % affine)
        del y
        for training in (0, 1):
            what = "bn_bwd affine=%s training=%d" % (affine, training)
            dx, dgam, dbet = Flat(m * n, cuda), Flat(n, cuda), Flat(n, cuda)
            wb = L.b2ctr_colstats_workspace_bytes(m, n)
            ws = _nan_workspace(wb, cuda)
            _check(L.b2ctr_bn_bwd(xb.buf.data_ptr(), meanf.buf.data_ptr(), varf.buf.data_ptr(), p(g_),
                                  dyf.buf.data_ptr(), dx.buf.data_ptr(), dgam.buf.data_ptr(), dbet.buf.data_ptr(), m, n,
                                  0.0, training, ws.data_ptr(), wb, st), "bn_bwd")
            for f, nm in ((dx, "dx"), (dgam, "dgamma"), (dbet, "dbeta")):
                f.check_outside(what + " " + nm)
            assert bool((ws[wb // 4:].view(torch.int32) == NAN_BITS).all()), what + ": wrote past its workspace"
            _same(dbet.values(), S1, what + " dbeta")
            _same(dgam.values(), S2, what + " dgamma")
            got = dx.values().reshape(m, n)
            if not training:
                _same(got, gm * rs * dy, what + " dx")
            else:
                A, Bt = S1 / m, xn * S2 / m
                want = gm * rs * (dy - A - Bt)
                if pow2m:
                    _same(got, want, what + " dx")
                else:
                    bound = 6 * 2.0 ** -24 * (gm * rs).abs() * (dy.abs() + A.abs() + Bt.abs())
                    err = (got.double() - want).abs()
                    assert bool((err <= bound).all()), "%s dx: %g ulp of its terms" % (
                        what, float((err / bound.clamp_min(1e-30)).max() * 6))
            del dx, ws
    frozen.check("bn")
    del xb, dyf

    # ---- Dice: p in {1/2, 0, 1}
    xd, ad, vd = _flat(o["x_d"], cuda), _flat(o["alpha"], cuda), _flat(o["var_d"], cuda)
    dyf = _flat(o["dy"], cuda)
    frozen = _freeze(xd.buf, ad.buf, vd.buf, dyf.buf, meanf.buf)
    rs = 1.0 / d64(o["var_d"]).sqrt()
    xn = (x64 - d64(o["mu"])) * rs
    assert bool(((xn == 0) | (xn.abs() >= GAP)).all())
    pr = torch.where(xn == 0, 0.5, (xn > 0).double())
    al = d64(o["alpha"])
    y = Flat(m * n, cuda)
    _check(L.b2ctr_dice_fwd(xd.buf.data_ptr(), meanf.buf.data_ptr(), vd.buf.data_ptr(), ad.buf.data_ptr(),
                            y.buf.data_ptr(), m, n, 0.0, st), "dice_fwd")
    y.check_outside("dice_fwd")
    _same(y.values().reshape(m, n), al * (1 - pr) * x64 + pr * x64, "dice_fwd")
    del y
    g = dy * x64 * (1 - al) * pr * (1 - pr)
    Sg, Sgx, Sa = g.sum(0), (g * xn).sum(0), (dy * x64 * (1 - pr)).sum(0)
    _fits(g.abs().sum(0), 2.0 ** -3, "dice sum g")
    _fits((dy * x64 * (1 - pr)).abs().sum(0), 0.5, "dice sum dy x (1 - p)")
    assert bool((Sgx == 0).all())                      # g is non-zero only where xn = 0
    dx1 = dy * (al + (1 - al) * pr)
    for training in (0, 1):
        what = "dice_bwd training=%d" % training
        dx, da = Flat(m * n, cuda), Flat(n, cuda)
        wb = L.b2ctr_dice_bwd_workspace_bytes(m, n)
        ws = _nan_workspace(wb, cuda)
        _check(L.b2ctr_dice_bwd(xd.buf.data_ptr(), meanf.buf.data_ptr(), vd.buf.data_ptr(), ad.buf.data_ptr(),
                                dyf.buf.data_ptr(), dx.buf.data_ptr(), da.buf.data_ptr(), m, n, 0.0, training,
                                ws.data_ptr(), wb, st), "dice_bwd")
        dx.check_outside(what + " dx")
        da.check_outside(what + " dalpha")
        assert bool((ws[wb // 4:].view(torch.int32) == NAN_BITS).all()), what + ": wrote past its workspace"
        _same(da.values(), Sa, what + " dalpha")
        # training: dx = dx1 + rs (g - fp32(Sg * fp32(1/m))); the xn * Sgx term is 0 exactly
        v = _round32(g - _round32(Sg * invm)) if training else g
        _same(dx.values().reshape(m, n), _round32(dx1 + rs * v), what + " dx")
        del dx, ws
    frozen.check("dice")


@pytest.mark.parametrize("n", BN_N)
@pytest.mark.parametrize("m", BN_M)
def test_batchnorm_and_dice_exact(cuda, m, n):
    """m around one 512-row block of the column reductions, n around the 256 threads of a block (they go round at
    n = 1300) and the 128 columns of each colsum_final CTA."""
    assert [-(-mm // STAT_ROWS) for mm in BN_M] == [1, 1, 1, 2, 2]
    _bn_dice_case(cuda, m, n, seed=m * 10 + n)


@pytest.mark.parametrize("m,n", BN_BIG, ids=["c4_n40", "c4_n129", "c4_plus_1_n1", "c4_plus_1_n257", "onn_bn"])
def test_batchnorm_and_dice_exact_at_bench_shapes(cuda, m, n):
    """DIN's Dice at C4 (B * T = 409,600 rows: 800 blocks), one row more (a block of one row), and ONN's
    BatchNormalization (65,536 x 1300)."""
    _bn_dice_case(cuda, m, n, seed=m + n)


# ================================================================================================ LayerNorm
LN_N = [1, 31, 32, 33, 64, 65, 128, 129, 256, 257, 512, 513, 1024]
LN_ROWS = [1, 7, 8, 9, LN_PASS - 1, LN_PASS, LN_PASS + 1]
LN_VARIANTS = {"plain": (False, False, False, False, False), "residual_affine": (True, True, True, True, True),
               "gamma_dgamma": (False, True, False, True, False), "residual_dbeta": (True, False, True, False, True)}


def _ln_rows(gen, rows, n):
    """x = mu + d per row: integer d with sum 0 and sum d^2 = n 4^(1 + k), k in 0..2 per row, shuffled, so the mean
    is mu and rstd is 2^-(1 + k) with eps = 0 (n = 1: d = 0, eps = 1)."""
    if n == 1:
        d0 = [0.0]
    elif n % 2 == 0:
        d0 = [2.0, -2.0] * (n // 2)
    else:
        d0 = [2.0, -2.0] * ((n - 5) // 2) + [3.0, -3.0, 1.0, -1.0, 0.0]
    d = torch.tensor(d0)[torch.argsort(torch.rand((rows, n), generator=gen), 1)]
    d *= 2.0 ** _ints(gen, (rows, 1), 0, 2)
    return _ints(gen, (rows, 1), -3, 3) + d


def _layernorm_case(cuda, rows, n, variant, seed):
    L, K = _lib(), _kern()
    use_b, use_g, use_beta, want_dg, want_db = LN_VARIANTS[variant]
    gen = torch.Generator().manual_seed(seed)
    eps = 1.0 if n == 1 else 0.0
    x = _ln_rows(gen, rows, n)
    a = _ints(gen, (rows, n), -4, 4) if use_b else x
    src = Window(rows, 2 * n + 9, 1, 2, n, n + 4, cuda)
    src.fill(torch.stack([a, x - a], 1).to(cuda))
    ap, bp = src.buf[:, 1:].data_ptr(), src.buf[:, 1 + n + 4:].data_ptr() if use_b else None
    gamma = _flat(torch.tensor([-2.0, -1.0, -0.5, 0.5, 1.0, 2.0])[torch.randint(0, 6, (n,), generator=gen)], cuda) \
        if use_g else None
    beta = _flat(_ints(gen, (n,), -5, 5) * 0.25, cuda) if use_beta else None
    p = lambda f: f.buf.data_ptr() if f is not None else None          # noqa: E731
    y = Window(rows, n + 6, 2, 1, n, n, cuda)
    stats = Flat(2 * rows, cuda)
    frozen = _freeze(src.buf, *[f.buf for f in (gamma, beta) if f is not None])
    st = K.stream()
    _check(L.b2ctr_layernorm_fwd(ap, src.ld, bp, src.ld, p(gamma), p(beta), y.buf[:, 2:].data_ptr(), y.ld,
                                 stats.buf.data_ptr(), rows, n, eps, st), "layernorm_fwd")
    y.check_outside("layernorm_fwd y")
    stats.check_outside("layernorm_fwd stats")
    # float32 restatement of the forward: mean by IEEE division, fma sum of squares, sqrtf, 1 / x, __fmul_rn, __fadd_rn
    x64 = _round32(a.to(cuda).double() + (x - a).to(cuda).double() if use_b else x.to(cuda).double())
    _fits(x64.abs().sum(1), 1.0, "layernorm sum")
    mean = _round32(x64.sum(1, keepdim=True) / n)
    dlt = _round32(x64 - mean)
    _fits((dlt * dlt).sum(1), 1.0, "layernorm sum of squares")
    rstd = _round32(1.0 / _round32(torch.sqrt(_round32(_round32((dlt * dlt).sum(1, keepdim=True) / n) + eps))))
    xh = _round32(dlt * rstd)
    gm = gamma.values().double() if use_g else None
    want = _round32(xh * gm) if use_g else xh
    want = _round32(want + beta.values().double()) if use_beta else want
    _same(stats.values().reshape(rows, 2), torch.cat([mean, rstd], 1), "layernorm stats")
    _same(y.values().reshape(rows, n), want, "layernorm_fwd y (%s)" % variant)
    assert bool(_pow2((1.0 / rstd).round().long()).all()) and torch.equal(rstd, 1.0 / (1.0 / rstd).round())
    # backward from a NaN-padded dy window into a dx window; the NaN workspace's partial rows are all written
    dyw = _put(rows, n + 3, 3, _ints(gen, (rows, n), -2, 2), cuda)
    dx = Window(rows, n + 5, 1, 1, n, n, cuda)
    dgam, dbet = Flat(n, cuda), Flat(n, cuda)
    nb = L.b2ctr_layernorm_bwd_workspace_bytes(rows, n)
    nblk = min(-(-rows // 8), 2 * NUM_SMS)
    assert nb == nblk * 8 * 2 * n * 4
    ws = _nan_workspace(nb, cuda)
    frozen_b = _freeze(dyw.buf, stats.buf)
    _check(L.b2ctr_layernorm_bwd(ap, src.ld, bp, src.ld, p(gamma), stats.buf.data_ptr(), dyw.buf[:, 3:].data_ptr(),
                                 dyw.ld, dx.buf[:, 1:].data_ptr(), dx.ld, dgam.buf.data_ptr() if want_dg else None,
                                 dbet.buf.data_ptr() if want_db else None, rows, n, ws.data_ptr(), nb, st),
           "layernorm_bwd")
    frozen.check("layernorm")
    frozen_b.check("layernorm_bwd")
    dx.check_outside("layernorm_bwd dx")
    wsi = ws.view(torch.int32)
    assert not bool((wsi[:nb // 4] == NAN_BITS).any()), "layernorm_bwd left partial rows of its workspace unwritten"
    assert bool((wsi[nb // 4:] == NAN_BITS).all()), "layernorm_bwd wrote past its workspace"
    g = dyw.values().reshape(rows, n).double()
    gg = g * gm if use_g else g
    _fits(gg.abs().sum(1) + (gg * xh).abs().sum(1), 2.0 ** -2, "layernorm row sums")
    got = dx.values().reshape(rows, n)
    if _pow2(torch.tensor(n)):
        _same(got, rstd * (gg - gg.mean(1, keepdim=True) - xh * (gg * xh).mean(1, keepdim=True)), "layernorm dx")
    else:
        # dx = rstd (gg - s1 - xh s2), s1 = S1 * inv_n, s2 = S2 * inv_n: each product may be contracted into the
        # subtraction that follows it (an fma), so dx is one of the four fp32 restatements
        inv_n = float(np.float32(1.0) / np.float32(n))
        S1, S2 = gg.sum(1, keepdim=True), (gg * xh).sum(1, keepdim=True)
        s2 = _round32(S2 * inv_n)
        gd, ok = got.double(), torch.zeros_like(got, dtype=torch.bool)
        for t in (_round32(gg - _round32(S1 * inv_n)), _round32(gg - S1 * inv_n)):
            for v in (_round32(t - xh * s2), _round32(t - _round32(xh * s2))):
                ok |= gd == _round32(rstd * v)
        assert bool(ok.all()), "layernorm dx (%s): %d entries match no fp32 restatement" % (variant, int((~ok).sum()))
    _fits((g * xh).abs().sum(0), 2.0 ** -3, "layernorm dgamma")
    for f, want_, on, nm in ((dgam, (g * xh).sum(0), want_dg, "dgamma"), (dbet, g.sum(0), want_db, "dbeta")):
        f.check_outside("layernorm_bwd " + nm)
        if on:
            _same(f.values(), want_, "layernorm " + nm)
        else:
            assert bool((f.buf.view(torch.int32) == NAN_BITS).all()), "layernorm_bwd wrote %s" % nm


@pytest.mark.parametrize("variant", sorted(LN_VARIANTS))
@pytest.mark.parametrize("rows", LN_ROWS, ids=["one", "seven", "cta", "cta_plus_1", "pass_minus_1", "pass",
                                               "pass_plus_1"])
@pytest.mark.parametrize("n", LN_N)
def test_layernorm_exact(cuda, n, rows, variant):
    """n: every NK instantiation (1, 2, 4, 8, 16, 32 lane rounds), full and with idle lanes; rows around one CTA
    and the backward's pass of 264 CTAs x 8 warps."""
    assert LN_PASS == 2112
    _layernorm_case(cuda, rows, n, variant, seed=rows * 1031 + n + len(variant))


@pytest.mark.parametrize("rows,n", [(409600, 64), (409601, 64), (409601, 129)],
                         ids=["bst", "bst_plus_1", "bst_plus_1_n129"])
def test_layernorm_exact_at_the_bst_shape(cuda, rows, n):
    """tools/bst_bench.py's rows, B * T = 8192 * 50, with its E = 64, and one row more."""
    _layernorm_case(cuda, rows, n, "residual_affine", seed=rows + n)


# ================================================================================================ ONN ffm_product
FFM_SHIFT = 28                 # floats between consecutive tables in the shared base: a multiple of 4 (16 bytes)
FFM_KINDS = ("i32", "i64", "strided", "hashed", "pooled")


def _hash_ids(raw, vocab, mask_zero):
    from oracle import farmhash
    lut = {int(u): farmhash.hash_bucket(int(u), vocab, mask_zero) for u in torch.unique(raw).tolist()}
    return torch.tensor([lut[int(v)] for v in raw.tolist()], dtype=torch.int64)


def _ffm_case(cuda, B, F, E, reduce_sum, seed, kinds=None, vocab=41, out_col=0, out_pad=4, oob=True):
    """Tables are overlapping windows of one base buffer (table a*F + c at a multiple of 28 floats), so a swapped
    table reads other values.  Field a's kind is kinds[a] (default: FFM_KINDS in turn).  Products into a column
    window of a NaN buffer, the gradient read from a NaN-padded window, per-lookup gradients into a NaN scratch."""
    from deepctr_b200 import _lib as Lm
    L, K = _lib(), _kern()
    gen = torch.Generator().manual_seed(seed)
    P = F * (F - 1) // 2
    kinds = kinds or [FFM_KINDS[a % len(FFM_KINDS)] for a in range(F)]
    base = _ints(gen, (F * F * FFM_SHIFT + vocab * E + 4,), -3, 3).to(cuda)
    ptrs = [base.data_ptr() + 4 * FFM_SHIFT * (a * F + c) if a != c else 0 for a in range(F) for c in range(F)]
    tables = torch.tensor(ptrs, dtype=torch.int64, device=cuda)
    rid = torch.full((B, F), -1, dtype=torch.int64)    # resolved row per (sample, id field), -1 out of range
    fields, keep, pooled, n_oob = [], [], {}, 0
    gw_ld = F * (F - 1) * E + 4
    gwin = Window(B, gw_ld, 0, F, (F - 1) * E, (F - 1) * E, cuda)
    for a, kind in enumerate(kinds):
        grad = gwin.buf[:, a * (F - 1) * E:]
        if kind == "pooled":
            pw = _put(B, (F - 1) * E + 8, 4, _ints(gen, (B, (F - 1) * E), -3, 3), cuda)
            pooled[a] = pw.values()[:, 0]
            keep.append(pw.buf)
            fields.append(K.ffm_field(pooled=pw.buf[:, 4:], grad=grad))
            continue
        if kind == "hashed":
            raw = torch.randint(0, 300, (B,), generator=gen)
            ids = _hash_ids(raw, vocab, a % 2 == 1)
            mode = Lm.HASH_FARM_MASK_ZERO if a % 2 == 1 else Lm.HASH_FARM
        else:
            raw = torch.randint(-3 if oob else 0, vocab + 3 if oob else vocab, (B,), generator=gen)
            ids, mode = raw.clone(), Lm.HASH_NONE
        ok = (ids >= 0) & (ids < vocab)
        n_oob += int((~ok).sum())
        rid[:, a] = torch.where(ok, ids, -1)
        dt = torch.int64 if kind in ("i64", "hashed") else torch.int32
        if kind == "strided":
            col = torch.full((B, 3), 7, dtype=dt)
            col[:, 1] = raw.to(dt)
            col = col.to(cuda)
            idx = col[:, 1]
        else:
            col = idx = raw.to(dt).to(cuda)
        keep.append(col)
        fields.append(K.ffm_field(idx=idx, vocab=vocab, hash_mode=mode, grad=grad))
    width = P * (1 if reduce_sum else E)
    ld = out_col + width + out_pad
    out = Window(B, ld, out_col, 1, width, width, cuda)
    frozen = _freeze(base, tables, *keep)
    K.embed_oob_count(reset=True)
    _check(L.b2ctr_ffm_product_fwd((Lm.FfmField * F)(*fields), F, tables.data_ptr(), E, int(reduce_sum),
                                   out.buf.data_ptr(), ld, out_col, B, K.stream()), "ffm_product_fwd")
    assert K.embed_oob_count(reset=True) == n_oob, "ffm_product_fwd: out-of-range ids miscounted"
    out.check_outside("ffm_product_fwd")
    g = _put(B, ld, out_col, _ints(gen, (B, width), -3, 3), cuda)
    frozen_g = _freeze(g.buf)
    _check(L.b2ctr_ffm_product_bwd((Lm.FfmField * F)(*fields), F, tables.data_ptr(), E, int(reduce_sum),
                                   g.buf.data_ptr(), ld, out_col, B, K.stream()), "ffm_product_bwd")
    assert K.embed_oob_count(reset=True) == 0, "ffm_product_bwd counted out-of-range ids"
    frozen.check("ffm_product")
    frozen_g.check("ffm_product_bwd")
    gwin.check_outside("ffm_product_bwd grad")
    # float64 reference over sample chunks
    iu, ju = torch.triu_indices(F, F, 1)
    e = torch.arange(E)
    got_out = out.values().reshape(B, P, -1)
    got_g = gwin.values().reshape(B, F, F - 1, E)
    chunk = max(1, (1 << 23) // (P * E))
    for b0 in range(0, B, chunk):
        sl = slice(b0, min(B, b0 + chunk))
        r = rid[sl]
        nb_ = r.shape[0]

        def operand(a_idx, c_idx):
            """[n, P, E]: field a_idx[p]'s operand for partner c_idx[p]."""
            ra = r[:, a_idx]
            off = (a_idx * F + c_idx) * FFM_SHIFT
            ix = (off[None, :] + ra.clamp_min(0) * E)[..., None] + e
            v = base[ix.to(cuda)].double() * (ra >= 0).to(cuda)[..., None]
            for a, pv in pooled.items():
                sel = (a_idx == a).nonzero().flatten()
                if len(sel):
                    s = c_idx[sel] - (c_idx[sel] > a).long()
                    v[:, sel.to(cuda)] = pv[sl].double().reshape(nb_, F - 1, E)[:, s.to(cuda)]
            return v
        ei, ej = operand(iu, ju), operand(ju, iu)
        prod = ei * ej
        _fits(prod.abs().sum(-1), 1.0, "ffm products")
        _same(got_out[sl], prod.sum(-1, keepdim=True) if reduce_sum else prod, "ffm_product_fwd")
        gp = g.values()[sl].double().reshape(nb_, P, -1)
        want = torch.empty((nb_, F, F - 1, E), dtype=torch.float64, device=cuda)
        want[:, iu.to(cuda), (ju - 1).to(cuda)] = gp * ej
        want[:, ju.to(cuda), iu.to(cuda)] = gp * ei
        _same(got_g[sl], want, "ffm_product_bwd")


@pytest.mark.parametrize("reduce_sum", [0, 1], ids=["elementwise", "reduce_sum"])
@pytest.mark.parametrize("E", [1, 3, 4, 5, 64])
@pytest.mark.parametrize("F", [2, 3, 32, 33, 64])
def test_ffm_product_exact_fields_and_dims(cuda, F, E, reduce_sum):
    """F = 33 and 64: the lanes resolve the ids in two rounds; P up to 2016 pairs (63 rounds of 32).  E = 4 and 64
    take the float4 path, 1 / 3 / 5 the scalar one.  Nine samples: two CTAs, the second with one warp."""
    _ffm_case(cuda, 9, F, E, reduce_sum, seed=100 * F + E + reduce_sum)


FFM_B = [1, 7, 8, 9, WARP_CAP - 1, WARP_CAP, WARP_CAP + 1, 65537]


@pytest.mark.parametrize("reduce_sum", [0, 1], ids=["elementwise", "reduce_sum"])
@pytest.mark.parametrize("F,E", [(3, 4), (33, 1)], ids=["F3_E4", "F33_E1"])
@pytest.mark.parametrize("B", FFM_B, ids=["one", "seven", "cta", "cta_plus_1", "cap_minus_1", "cap", "cap_plus_1",
                                          "b65537"])
def test_ffm_product_exact_at_block_and_grid_boundaries(cuda, B, F, E, reduce_sum):
    """One warp per sample, 8 a CTA, grid_for(B, 8, 8) = 1056 CTAs: past 8,448 samples a warp reuses its shared
    id slots for a second sample."""
    assert WARP_CAP == 8448
    _ffm_case(cuda, B, F, E, reduce_sum, seed=B + F + reduce_sum)


@pytest.mark.parametrize("reduce_sum", [0, 1], ids=["elementwise", "reduce_sum"])
@pytest.mark.parametrize("out_col,out_pad", [(1, 3), (0, 3)], ids=["odd_column", "odd_pitch"])
def test_ffm_product_scalar_path_with_e_a_multiple_of_4(cuda, out_col, out_pad, reduce_sum):
    """E = 8 with an output column or pitch that is not a multiple of 4: the scalar path."""
    F, E = 5, 8
    width = F * (F - 1) // 2 * (1 if reduce_sum else E)
    assert (out_col + width + out_pad) % 4 or out_col % 4
    _ffm_case(cuda, 133, F, E, reduce_sum, seed=out_col + reduce_sum, out_col=out_col, out_pad=out_pad)


@pytest.mark.parametrize("reduce_sum", [0, 1], ids=["elementwise", "reduce_sum"])
def test_ffm_product_onn_bench_shape(cuda, reduce_sum):
    """tools/onn_bench.py: 26 fields of 1M ids, E = 4, B = 65,536, int32 ids in range."""
    _ffm_case(cuda, 65536, 26, 4, reduce_sum, seed=26 + reduce_sum, kinds=["i32"] * 26, vocab=1 << 20, oob=False)


class _Emb(object):
    def __init__(self, t):
        self.t = t

    def materialize(self):
        return self.t


class _Table(object):
    def __init__(self, t):
        self.embeddings = _Emb(t)


def test_field_aware_plan_refuses_misaligned_tables(cuda):
    """b2ctr_ffm_product_* take the float4 path for E % 4 == 0 from the other operands' alignment: a table that is
    not 16-byte aligned is refused on the host, before anything is launched."""
    from deepctr_b200 import _lib as Lm
    from deepctr_b200.inputs import FieldAwarePlan
    F = 3
    buf = torch.zeros(F * F * 64 + 8, device=cuda)

    def plan(E, shift):
        tabs = [None if a == c else _Table(buf[shift + (a * F + c) * 64:][:32]) for a in range(F) for c in range(F)]
        fields = [("f%d" % a, 1, Lm.POOL_NONE, Lm.HASH_NONE, 8) for a in range(F)]
        return FieldAwarePlan(fields, tabs, E, False, [], [], [])
    torch.cuda.synchronize()
    before = Lm.launch_count()
    for shift in (1, 2, 3):
        with pytest.raises(ValueError, match="16-byte aligned"):
            plan(4, shift)._table_array(cuda)
    assert Lm.launch_count() == before
    for E, shift in ((4, 0), (4, 4), (5, 1), (3, 2)):      # aligned, or a dim the float4 path never takes
        assert plan(E, shift)._table_array(cuda).shape == (F * F,)


# ================================================================================================ tolerance companions
@pytest.mark.parametrize("m,n", [(409600, 40), (409601, 80), (65536, 1300)], ids=["c4", "c4_plus_1", "onn_bn"])
def test_batchnorm_and_dice_random_data_at_bench_shapes(cuda, m, n):
    """Random data, the real eps (1e-3 BatchNormalization, 1e-9 Dice), test_simt_kernels_gpu's bounds."""
    SIMT.test_dice_and_batchnorm_match_float64(cuda, m, n)


@pytest.mark.parametrize("B,T,E", [(8192, 50, 64), (THREAD_CAP // 64 + 1, 7, 64), (2 * WARP_CAP + 1, 65, 3)])
def test_din_random_data_at_bench_shapes(cuda, B, T, E):
    SIMT.test_din_attention_input_matches_float64(cuda, B, T, E)
    SIMT.test_din_pool_matches_float64(cuda, B, T, E)


@pytest.mark.parametrize("rows,n", [(409601, 64), (LN_PASS + 1, 513), (LN_PASS + 1, 1024)])
def test_layernorm_random_data_at_bench_shapes(cuda, rows, n):
    """Random data, eps 1e-9, test_bst_gpu's tolerances, with the residual and gamma / beta."""
    got, want, _ = BST._ln_case(cuda, rows, n, True, True, seed=rows + n)
    for k, (name, tol) in enumerate((("y", 1e-5), ("dx", 1e-4), ("dgamma", 1e-5), ("dbeta", 1e-5))):
        BST._close(got[k], want[k], name, tol=tol)
