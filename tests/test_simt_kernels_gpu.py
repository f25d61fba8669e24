"""GPU: the SIMT kernels behind Dice / BatchNormalization, DIN attention pooling, sequence pooling and weighting,
AutoInt's InteractingLayer and the vector CrossNet, called directly through deepctr_b200.kernels and compared with a
float64 torch restatement of the same operation (include/b2ctr.h and the kernel comments).

The shapes reach the branches the layer tests never do: column statistics over many 512-row blocks (m = 102 400
is the C4 shape B*T of DIN's Dice layers) and more than 256 columns, bags longer than a warp, empty bags, every
position masked, ties in max pooling, up to 64 AutoInt fields and 32-wide heads, CrossNet rows wider than a
warp.  Batches are not a multiple of a CTA's 8 warps, one batch per kernel makes the grid-stride loops go round
more than once, and every input that has a pitch is a window of a wider buffer that is checked to be unchanged.

Tolerances: kernels that round each result once are compared bit for bit with the fp32 rounding of the float64
value; a sum of n terms may differ by (depth) * 2^-23 * sum|terms|, depth being the longest chain of additions in
the kernel's order; everything else is compared normwise, max|got - ref| / max|ref| < 2e-5, as the AFM tests do.
The two masking constants of the reference are computed in fp32 as the reference does: x - 1e9 of max pooling
(its ulp at 1e9 is 64, so masked entries with |x| < 32 tie) and the softmax padding -2^32 + 1 (= -2^32 in fp32).
"""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

U = 2.0 ** -24                                  # unit roundoff of fp32
STAT_ROWS = 512                                 # rows per block of the column reductions (kStatRows)
NEG_PAD = float(np.float32(-4294967295.0))      # -2^32 + 1 in fp32 (= -2^32)


def _kern():
    from deepctr_b200 import kernels as K, _lib as L
    return K, L


def _normwise(got, ref, what, tol=2e-5, dim=None, mag=None):
    """max|got - ref| / max|ref| < tol, over the whole tensor or per slice along `dim` (per column with dim=0).
    `mag`, when given, replaces |ref| in the scale: the summed magnitudes of the terms of a formula whose result
    may cancel (with a single row, a column's scale is that row's)."""
    ref = ref.detach().double()
    err = (got.double() - ref).abs()
    mag = ref.abs() if mag is None else mag.detach().double()
    if dim is None:
        err, scale = err.max(), mag.max()
    else:
        err, scale = err.amax(dim=dim), mag.amax(dim=dim)
    worst = float((err / scale.clamp_min(1e-30)).max())
    assert worst < tol, "%s: max error %.3e relative to max |value|" % (what, worst)


def _sum_close(got, ref, abs_sum, depth, what):
    """A sum whose longest addition chain is `depth`: |got - ref| <= (depth + 8) * 2^-23 * sum|terms|."""
    err = (got.double() - ref.detach().double()).abs()
    bound = (depth + 8) * 2 * U * abs_sum.detach().double() + 1e-37
    worst = float((err / bound).max())
    assert worst <= 1.0, "%s: error %.3g times the summation bound" % (what, worst)


def _fp32_exact(got, ref, what):
    """One fp32 rounding of a result that is exact in float64."""
    assert torch.equal(got, ref.detach().float()), "%s differs from the fp32 rounding of the float64 value" % what


def _rand(gen, shape, dev, std=1.0, mean=0.0):
    return torch.randn(shape, generator=gen, device=dev, dtype=torch.float32) * std + mean


def _window(gen, rows, cols, tail, dev, std=1.0):
    """[rows, cols] as the leading columns of a [rows, cols + tail] buffer; returns (buffer, window, its copy)."""
    buf = _rand(gen, (rows, cols + tail), dev, std)
    return buf, buf[:, :cols], buf.clone()


# ================================================================================================
# Dice / BatchNormalization: colstats, moving_update, bn_apply / bn_bwd, dice_fwd / dice_bwd
# ================================================================================================
def _stat_depth(m):
    return min(m, STAT_ROWS) + -(-m // STAT_ROWS)


def _batch_stats(x64, mean_k, var_k):
    """The batch mean / biased variance in float64, valued at the kernel's statistics (checked against float64
    separately) so that each kernel is measured on its own error; the gradient flows through the batch
    statistics as in training."""
    mu = x64.mean(dim=0)
    var = ((x64 - mu) ** 2).mean(dim=0)
    return mu + (mean_k.double() - mu).detach(), var + (var_k.double() - var).detach()


@pytest.mark.parametrize("n", [1, 40, 80, 300])
@pytest.mark.parametrize("m", [1, 511, 512, 513, 102400])
def test_dice_and_batchnorm_match_float64(cuda, m, n):
    K, L = _kern()
    gen = torch.Generator(device=cuda).manual_seed(1000 * n + m % 997)
    # columns of different scale and offset; column 0 has mean 100 and std 1, which a one-pass variance
    # (E[x^2] - E[x]^2 in fp32) would lose entirely
    x = _rand(gen, (m, n), cuda) * (0.5 + 1.5 * torch.rand(n, generator=gen, device=cuda)) \
        + _rand(gen, (n,), cuda, 2.0)
    x[:, 0] = _rand(gen, (m,), cuda, 1.0, 100.0)
    dy = _rand(gen, (m, n), cuda)
    x64 = x.double()

    # ---- column statistics (two passes over ceil(m / 512) blocks) and the moving-average update
    stats = K.colstats(x, n, m, n)
    mean64 = x64.mean(dim=0)
    var64 = ((x64 - mean64) ** 2).mean(dim=0)
    depth = _stat_depth(m)
    _sum_close(stats[0], mean64, x64.abs().mean(dim=0), depth + 1, "colstats mean")
    # the variance is a sum of squared deviations from the fp32 mean: its error adds the squared mean error
    mean_err = (stats[0].double() - mean64).abs()
    err = (stats[1].double() - var64).abs() - mean_err ** 2
    assert float((err / ((depth + 12) * 2 * U * var64 + 1e-37)).max()) <= 1.0, "colstats variance"
    moving = _rand(gen, (2, n), cuda)
    mom = float(np.float32(0.99))
    want = moving.double() * mom + stats.double() * (1 - mom)       # 1 - mom is exact in fp32
    K.moving_update(moving, stats, mom)
    _normwise(moving, want, "moving_update", tol=8 * U, dim=1)

    gamma = 1.0 + _rand(gen, (n,), cuda, 0.3)
    beta = _rand(gen, (n,), cuda, 0.5)
    alpha = _rand(gen, (n,), cuda, 0.5)
    run_mean, run_var = _rand(gen, (n,), cuda), 0.5 + torch.rand(n, generator=gen, device=cuda)
    for training in (0, 1):
        mean, var = (stats[0].contiguous(), stats[1].contiguous()) if training else (run_mean, run_var)
        tag = "training" if training else "inference"

        # ---- BatchNormalization (Keras eps 1e-3), gamma / beta as tensors and as NULL
        for g_, b_ in ((gamma, beta), (None, None)):
            what = "bn %s %s" % (tag, "affine" if g_ is not None else "plain")
            xr = x64.clone().requires_grad_(True)
            g64 = (g_ if g_ is not None else torch.ones_like(gamma)).double().requires_grad_(True)
            b64 = (b_ if b_ is not None else torch.zeros_like(beta)).double().requires_grad_(True)
            mu, va = _batch_stats(xr, mean, var) if training else (mean.double(), var.double())
            xn = (xr - mu) / torch.sqrt(va + np.float32(1e-3))
            ref = xn * g64 + b64
            (ref * dy.double()).sum().backward()
            y = K.bn_apply(x, mean, var, g_, b_, m, n, 1e-3)
            _normwise(y, ref, what + " y", dim=0, mag=(xn * g64).abs() + b64.abs())
            dx, dgamma, dbeta = K.bn_bwd(x, mean, var, g_, dy, m, n, 1e-3, training)
            # dx = gamma rs (dy - mean(dy) - xn mean(dy xn)) in training, gamma rs dy in inference
            a, xa = dy.double().abs(), xn.detach().abs()
            mag = (g64 / torch.sqrt(va + np.float32(1e-3))).abs() * (a + a.mean(dim=0) + xa * (a * xa).mean(dim=0))
            _normwise(dx, xr.grad, what + " dx", dim=0, mag=mag)
            _sum_close(dbeta, b64.grad, dy.double().abs().sum(dim=0), depth, what + " dbeta")
            _sum_close(dgamma, g64.grad, (dy.double() * xn.detach()).abs().sum(dim=0), depth + 4, what + " dgamma")

        # ---- Dice (eps 1e-9): p = sigmoid(xn), y = alpha (1 - p) x + p x
        xr = x64.clone().requires_grad_(True)
        a64 = alpha.double().requires_grad_(True)
        mu, va = _batch_stats(xr, mean, var) if training else (mean.double(), var.double())
        rs = 1 / torch.sqrt(va + np.float32(1e-9))
        xn = (xr - mu) * rs
        p = torch.sigmoid(xn)
        ref = a64 * (1 - p) * xr + p * xr
        (ref * dy.double()).sum().backward()
        y = K.dice_fwd(x, mean, var, alpha, m, n, 1e-9)
        a, xa, al = dy.double().abs(), xn.detach().abs(), alpha.double().abs()
        _normwise(y, ref, "dice %s y" % tag, dim=0, mag=x64.abs() * (al + 1))
        dx, dalpha = K.dice_bwd(x, mean, var, alpha, dy, m, n, 1e-9, training)
        # dx = dy (alpha + (1 - alpha) p) + rs (g - [training](mean(g) + xn mean(g xn))), g = dy x (1-alpha) p (1-p)
        g = (a * x64.abs() * (1 + al) * (p * (1 - p)).detach())
        mag = a * (al + 1) + rs.detach() * (g + g.mean(dim=0) + xa * (g * xa).mean(dim=0))
        _normwise(dx, xr.grad, "dice %s dx" % tag, dim=0, mag=mag)
        # the terms dy x (1 - p): 1 - p carries the absolute rounding of p, so the bound is taken on |dy x|
        _sum_close(dalpha, a64.grad, (a * x64.abs()).sum(dim=0), depth + 8, "dice %s dalpha" % tag)


def test_colstats_reads_a_window(cuda):
    """ld > n: the statistics of a column window of a wider buffer; the buffer is left as it was."""
    K, L = _kern()
    gen = torch.Generator(device=cuda).manual_seed(7)
    m, n = 1537, 300
    buf, xw, _ = _window(gen, m, n, 45, cuda)
    buf[:, n:] += 1e6                             # columns outside the window would show in the statistics
    before = buf.clone()
    stats = K.colstats(buf, buf.stride(0), m, n)
    x64 = xw.double()
    mean64 = x64.mean(dim=0)
    depth = _stat_depth(m)
    _sum_close(stats[0], mean64, x64.abs().mean(dim=0), depth + 1, "window mean")
    var64 = ((x64 - mean64) ** 2).mean(dim=0)
    err = (stats[1].double() - var64).abs() - (stats[0].double() - mean64) ** 2
    assert float((err / ((depth + 12) * 2 * U * var64)).max()) <= 1.0, "window variance"
    assert torch.equal(buf, before)


# ================================================================================================
# DIN: din_att_input_fwd / _bwd, din_pool_fwd / _bwd
# ================================================================================================
def _din_inputs(gen, B, T, E, dev):
    qbuf, q, _ = _window(gen, B, E, 5, dev)
    kbuf, k, _ = _window(gen, B, T * E, 11, dev, 0.5)
    lens = torch.randint(0, T + 1, (B,), generator=gen, device=dev)
    lens[0], lens[1 % B] = 0, T                   # an empty and a full history
    mask = (torch.arange(T, device=dev)[None, :] < lens[:, None]).to(torch.uint8)
    return qbuf, q, kbuf, k, mask


DIN_SHAPES = [(203, T, E) for T in (1, 7, 50, 200) for E in (1, 8, 64, 100)] + [(9001, 7, 8)]


@pytest.mark.parametrize("B,T,E", DIN_SHAPES)
def test_din_attention_input_matches_float64(cuda, B, T, E):
    K, L = _kern()
    gen = torch.Generator(device=cuda).manual_seed(B + 31 * T + E)
    qbuf, q, kbuf, k, _ = _din_inputs(gen, B, T, E, cuda)
    qb, kb = qbuf.clone(), kbuf.clone()
    out = K.din_att_input_fwd(q, qbuf.stride(0), k, kbuf.stride(0), B, T, E)
    q64 = q.double().reshape(B, 1, E).requires_grad_(True)
    k64 = k.double().reshape(B, T, E).requires_grad_(True)
    qr = q64.expand(B, T, E)
    ref = torch.cat([qr, k64, qr - k64, qr * k64], dim=-1)
    _fp32_exact(out, ref, "[q, k, q-k, q*k]")          # one rounding per element, exact in float64
    g = _rand(gen, (B, T, 4 * E), cuda)
    (ref * g.double()).sum().backward()
    dq, dk = K.din_att_input_bwd(q, qbuf.stride(0), k, kbuf.stride(0), g, B, T, E)
    g64 = g.double()
    _sum_close(dq, q64.grad, (g64[..., :E].abs() + g64[..., 2 * E:3 * E].abs()
                              + (g64[..., 3 * E:] * k64.detach()).abs()).sum(dim=1, keepdim=True), 3 * T, "dq")
    gk_terms = g64[..., E:2 * E].abs() + g64[..., 2 * E:3 * E].abs() + (g64[..., 3 * E:] * q64.detach()).abs()
    _sum_close(dk, k64.grad, gk_terms, 3, "dkeys")
    assert torch.equal(qbuf, qb) and torch.equal(kbuf, kb)


def _ref_din_pool(score64, k64, mask, weight_norm, return_score):
    """AttentionSequencePoolingLayer tail (sequence.py:278-291) in float64; the padding is the fp32 -2^32."""
    valid = mask.bool()
    pad = torch.full_like(score64, NEG_PAD) if weight_norm else torch.zeros_like(score64)
    w = torch.where(valid, score64, pad)
    if weight_norm:
        w = torch.softmax(w, dim=-1)
    return w, (w if return_score else torch.einsum("bt,bte->be", w, k64))


@pytest.mark.parametrize("B,T,E", DIN_SHAPES)
def test_din_pool_matches_float64(cuda, B, T, E):
    K, L = _kern()
    gen = torch.Generator(device=cuda).manual_seed(7 * B + T + 13 * E)
    _, _, kbuf, k, mask = _din_inputs(gen, B, T, E, cuda)
    kb = kbuf.clone()
    ldk = kbuf.stride(0)
    score = _rand(gen, (B, T), cuda, 2.0)
    empty = mask.sum(dim=1) == 0
    for weight_norm in (0, 1):
        for return_score in (0, 1):
            what = "weight_norm=%d return_score=%d" % (weight_norm, return_score)
            out, w = K.din_pool_fwd(score, k, ldk, mask, B, T, E, weight_norm, return_score)
            s64 = score.double().requires_grad_(True)
            k64 = k.double().reshape(B, T, E).requires_grad_(True)
            w64, ref = _ref_din_pool(s64, k64, mask, weight_norm, return_score)
            if weight_norm:
                _normwise(w, w64, what + " weights", tol=(T + 16) * U)
                # every position masked: the softmax of T equal paddings
                assert torch.equal(w[empty], torch.full_like(w[empty], float(np.float32(1.0) / np.float32(T))))
            else:
                _fp32_exact(w, w64, what + " weights")
            if return_score:
                assert torch.equal(out.reshape(B, T), w)
            else:
                _sum_close(out.reshape(B, E), ref, torch.einsum("bt,bte->be", w64.abs(), k64.abs()),
                           2 * T + 16, what + " out")
            dout = _rand(gen, tuple(out.shape), cuda)
            (ref * dout.double().reshape(ref.shape)).sum().backward()
            dscore, dkeys = K.din_pool_bwd(w, k, ldk, mask, dout, B, T, E, weight_norm, return_score)
            dscore = dscore.reshape(B, T)
            assert bool((dscore[mask == 0] == 0).all()), what + ": masked positions must get dscore 0"
            _normwise(dscore, s64.grad, what + " dscore")
            if not return_score:
                _normwise(dkeys.reshape(B, T, E), k64.grad, what + " dkeys")
            else:
                assert dkeys is None
    assert torch.equal(kbuf, kb)


# ================================================================================================
# Sequence pooling / weighting: seqpool_fwd / _bwd, seqweight, seqscale
# ================================================================================================
def _bags(gen, B, T, E, dev):
    """[B, T, E] rows gathered from a small table: every other bag draws from 3 rows, so max pooling ties."""
    table = _rand(gen, (40, E), dev)
    ids = torch.randint(0, 40, (B, T), generator=gen, device=dev)
    ids[::2] = torch.randint(0, 3, (B // 2 + B % 2, T), generator=gen, device=dev)
    x = table[ids].contiguous()
    lens = torch.randint(0, T + 1, (B,), generator=gen, device=dev).to(torch.int32)
    lens[0], lens[1] = 0, T
    return x, lens


@pytest.mark.parametrize("E", [1, 64, 130])
@pytest.mark.parametrize("T", [1, 50, 200])
@pytest.mark.parametrize("validity", ["mask", "length"])
@pytest.mark.parametrize("mode", ["sum", "mean", "max"])
def test_seqpool_matches_float64(cuda, mode, validity, T, E):
    K, L = _kern()
    gen = torch.Generator(device=cuda).manual_seed(T * 1000 + E)
    B = 3001 if T * E < 10000 else 307        # 3001 * 130 (b, e) threads need more than one grid-stride pass
    x, lens = _bags(gen, B, T, E, cuda)
    valid = torch.arange(T, device=cuda)[None, :] < lens[:, None]
    if validity == "mask":
        # a mask that is not a prefix: validity from the mask alone
        valid = torch.rand((B, T), generator=gen, device=cuda) < 0.7
        valid[0] = False
        mask, length = valid.to(torch.uint8), None
    else:
        mask, length = None, lens
    code = L.POOL_BY_NAME[mode]
    out = K.seqpool_fwd(x, mask, length, B, T, E, code)
    x64 = x.double().requires_grad_(True)
    v3 = valid[:, :, None]
    if mode == "max":
        # x - 1e9 in fp32 as the reference computes it; the gradient of the subtraction is 1
        hist32 = torch.where(v3, x, x - 1e9)
        hist = x64 + (hist32.double() - x64).detach()
        ref = hist.amax(dim=1)                         # ties share the gradient evenly, as TF's reduce_max
        _fp32_exact(out.reshape(B, E), ref, "max pool")
    else:
        ref = (x64 * v3).sum(dim=1)
        terms = (x64.detach() * v3).abs().sum(dim=1)
        if mode == "mean":
            Lf = valid.sum(dim=1, keepdim=True).double()
            ref = ref / (Lf + 1e-8)
            terms = terms / (Lf + 1e-8)
        _sum_close(out.reshape(B, E), ref, terms, T + 2, "%s pool" % mode)
    dout = _rand(gen, (B, 1, E), cuda)
    (ref * dout.double().reshape(B, E)).sum().backward()
    dx = K.seqpool_bwd(x, mask, length, dout, B, T, E, code)
    # one rounding per element (g, g / (L + 1e-8) or g / cnt): within an ulp of float64
    assert float(((dx.double() - x64.grad).abs() - 2 * U * x64.grad.abs()).max()) <= 0, "%s pool dx" % mode
    if mode == "max":
        ties = (hist32 == hist32.amax(dim=1, keepdim=True)).sum(dim=1)
        assert T == 1 or int((ties > 1).sum()) > 0, "the inputs must contain ties"
        # an empty bag: every masked x - 1e9 rounds to -1e9, so the gradient is spread over all T positions
        if T > 1 and bool((x[0].abs() < 32).all()):
            assert torch.equal(dx[0], (dout[0].double() / T).float().expand(T, E))


@pytest.mark.parametrize("T", [1, 7, 50, 200])
@pytest.mark.parametrize("validity", ["mask", "length"])
def test_seqweight_and_seqscale_match_float64(cuda, validity, T):
    K, L = _kern()
    gen = torch.Generator(device=cuda).manual_seed(T + 5)
    B, E = 1201, 9
    w = _rand(gen, (B, T), cuda, 2.0)
    lens = torch.randint(0, T + 1, (B,), generator=gen, device=cuda).to(torch.int32)
    lens[0], lens[1] = 0, T
    valid = torch.arange(T, device=cuda)[None, :] < lens[:, None]
    if validity == "mask":
        valid = torch.rand((B, T), generator=gen, device=cuda) < 0.6
        valid[0] = False
        mask, length = valid.to(torch.uint8), None
    else:
        mask, length = None, lens
    empty = ~valid.any(dim=1)
    assert bool(empty.any())
    raw = K.seqweight(w, mask, length, B, T, 0)
    _fp32_exact(raw, torch.where(valid, w.double(), torch.zeros_like(w.double())), "raw weights")
    soft = K.seqweight(w, mask, length, B, T, 1)
    ref = torch.softmax(torch.where(valid, w.double(), torch.full_like(w.double(), NEG_PAD)), dim=1)
    _normwise(soft, ref, "softmax weights", tol=(T + 16) * U)
    assert torch.equal(soft[empty], torch.full_like(soft[empty], float(np.float32(1.0) / np.float32(T))))
    x = _rand(gen, (B, T, E), cuda)
    out = K.seqscale(x, soft, B * T, E)
    _fp32_exact(out, x.double() * soft.double()[:, :, None], "seqscale")


# ================================================================================================
# AutoInt: interacting_fwd / _bwd
# ================================================================================================
INT_MAX_FHD = 3072


def _ref_interacting(q, k, v, res, F, H, D, scaling):
    B = q.shape[0]
    qh, kh, vh = (t.reshape(B, F, H, D).transpose(1, 2) for t in (q, k, v))      # [B, H, F, D]
    s = qh @ kh.transpose(-1, -2)
    if scaling:
        s = s / np.sqrt(D)
    o = (torch.softmax(s, dim=-1) @ vh).transpose(1, 2).reshape(B, F, H * D)
    return o + res if res is not None else o


INT_SHAPES = [(F, H, D) for F in (1, 2, 26, 64) for H in (1, 2, 8) for D in (1, 3, 8, 32) if F * H * D <= INT_MAX_FHD]


@pytest.mark.parametrize("F,H,D", INT_SHAPES)
def test_interacting_matches_float64(cuda, F, H, D):
    K, L = _kern()
    gen = torch.Generator(device=cuda).manual_seed(F * 100 + H * 10 + D)
    B = 203
    q, k, v = (_rand(gen, (B, F, H * D), cuda, 1.0 / D ** 0.25) for _ in range(3))
    for scaling in (0, 1):
        for use_res in (False, True):
            what = "scaling=%d res=%d" % (scaling, use_res)
            # relu clamps part of the outputs: a residual centred below 0, or without one, v shifted by -1 in
            # odd samples and +1 in even ones (the attention output is a convex combination of the rows of v)
            res = _rand(gen, (B, F, H * D), cuda, 0.5, -0.2) if use_res else None
            sign = 1.0 - 2.0 * (torch.arange(B, device=cuda) % 2).float()
            vv = v if use_res else v + sign[:, None, None]
            out = K.interacting_fwd(q, k, vv, res, B, F, H, D, scaling)
            args = [t.double().requires_grad_(True) for t in (q, k, vv)]
            r64 = res.double().requires_grad_(True) if use_res else None
            pre = _ref_interacting(*args, r64, F, H, D, scaling)
            _normwise(out, torch.relu(pre), what + " out")
            zero = out == 0
            assert bool(zero.any()) and bool((~zero).any()), "relu must clamp some outputs and pass others"
            dout = _rand(gen, (B, F, H * D), cuda)
            # the float64 gradient takes relu' where the kernel's output is positive
            pre.backward(torch.where(zero, torch.zeros_like(dout), dout).double())
            dq, dk, dv, dres = K.interacting_bwd(q, k, vv, out, dout, use_res, B, F, H, D, scaling)
            for name, got, ref in (("dq", dq, args[0].grad), ("dk", dk, args[1].grad), ("dv", dv, args[2].grad)):
                _normwise(got, ref, "%s %s" % (what, name))
            if use_res:
                assert bool((dres[zero] == 0).all()), "dres must be 0 exactly where out is 0"
                assert torch.equal(dres[~zero], dout[~zero])
            else:
                assert dres is None


@pytest.mark.parametrize("F,H,D", [(65, 1, 8), (8, 1, 33), (64, 2, 32), (26, 8, 32), (64, 4, 13)])
def test_interacting_rejects_unsupported_shapes(cuda, F, H, D):
    """F > 64, d > 32 or F*H*d > 3072 (the backward's K, V, dK, dV in 48 KB of shared memory) are argument errors of
    both entry points, raised before any launch; F*H*d = 3072 runs forward and backward."""
    K, L = _kern()
    B = 3
    q = torch.zeros((B, F, H * D), device=cuda)
    n0 = L.launch_count()
    with pytest.raises(ValueError):
        K.interacting_fwd(q, q, q, q, B, F, H, D, 1)
    with pytest.raises(ValueError):
        K.interacting_bwd(q, q, q, q, q, True, B, F, H, D, 1)
    assert L.launch_count() == n0


def test_interacting_largest_shape_trains(cuda):
    K, L = _kern()
    gen = torch.Generator(device=cuda).manual_seed(3)
    B, F, H, D = 37, 64, 3, 16
    assert F * H * D == INT_MAX_FHD
    q, k, v, res = (_rand(gen, (B, F, H * D), cuda, 0.5) for _ in range(4))
    out = K.interacting_fwd(q, k, v, res, B, F, H, D, 1)
    args = [t.double().requires_grad_(True) for t in (q, k, v)]
    pre = _ref_interacting(*args, res.double(), F, H, D, True)
    _normwise(out, torch.relu(pre), "out")
    dout = _rand(gen, (B, F, H * D), cuda)
    pre.backward(torch.where(out == 0, torch.zeros_like(dout), dout).double())
    dq, dk, dv, _ = K.interacting_bwd(q, k, v, out, dout, True, B, F, H, D, 1)
    for name, got, ref in (("dq", dq, args[0].grad), ("dk", dk, args[1].grad), ("dv", dv, args[2].grad)):
        _normwise(got, ref, name)


# ================================================================================================
# CrossNet (vector): cross_vector_fwd / _bwd
# ================================================================================================
@pytest.mark.parametrize("B", [1, 1001, 9001])
@pytest.mark.parametrize("dim", [1, 7, 32, 33, 845])
def test_cross_vector_matches_float64(cuda, dim, B):
    K, L = _kern()
    gen = torch.Generator(device=cuda).manual_seed(dim * 10 + B)
    b0, x0, c0 = _window(gen, B, dim, 13, cuda)
    bl, xl, cl = _window(gen, B, dim, 6, cuda)
    w = _rand(gen, (dim,), cuda, 1.0 / np.sqrt(dim))
    bias = _rand(gen, (dim,), cuda, 0.3)
    out, s = K.cross_vector_fwd(x0, b0.stride(0), xl, bl.stride(0), w, bias, B, dim)
    x064, xl64 = x0.double().requires_grad_(True), xl.double().requires_grad_(True)
    w64 = w.double()
    s64 = xl64 @ w64
    ref = x064 * s64[:, None] + bias.double() + xl64
    s_terms = (xl64.detach() * w64).abs().sum(dim=1)
    _sum_close(s, s64, s_terms, dim, "s = <xl, w>")
    # out = x0 * s + bias + xl: the error of s scaled by |x0|, plus three roundings
    err = (out.double() - ref.detach()).abs()
    bound = x064.detach().abs() * ((dim + 8) * 2 * U * s_terms)[:, None] \
        + 4 * U * ((x064 * s64[:, None]).abs() + bias.double().abs() + xl64.abs()).detach()
    assert bool((err <= bound).all()), "out"
    dout = _rand(gen, (B, dim), cuda)
    (ref * dout.double()).sum().backward()
    dx0, dxl, ds = K.cross_vector_bwd(x0, b0.stride(0), w, dout, s, B, dim)
    ds64 = (dout.double() * x064.detach()).sum(dim=1)
    ds_terms = (dout.double() * x064.detach()).abs().sum(dim=1)
    _sum_close(ds, ds64, ds_terms, dim, "ds = <dout, x0>")
    # the float64 gradient of x0 is taken at the kernel's s (the value the backward is given)
    _fp32_exact(dx0, dout.double() * s.double()[:, None], "dx0")
    bound = w64.abs() * ((dim + 8) * 2 * U * ds_terms)[:, None] + 2 * U * (dout.double().abs()
                                                                          + (w64 * ds64[:, None]).abs())
    assert bool(((dxl.double() - xl64.grad).abs() <= bound).all()), "dxl"
    assert torch.equal(b0, c0) and torch.equal(bl, cl)
