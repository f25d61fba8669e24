"""GPU: the generated-operand split-bf16 GEMMs behind xDeepFM's CIN and DIN's first attention layer, the CIN fold and
the CIN helper kernels, called directly through deepctr_b200.kernels and compared with a float64 torch restatement of
the same operation (include/b2ctr.h and the kernel comments), run on the device so that production row counts
stay cheap.

Shapes: the CIN at the C3 benchmark shape (B = 32768 samples of 26 fields x 16, rows = B*D = 524 288; layer 0 has
h = m = 26 hidden maps padded to hp = 32, layer 1 has h = 64), DIN's first LocalActivationUnit layer at the C4 shape
(B = 8192, T = 50, E = 64, n = 80, rows = 409 600), and the edges the layers never reach: hp = 128 / 192 / 256 (the
j-block-major k-block walk of the forward), one and two N tiles, row counts that are not a multiple of the 128-row
tile, split-K slices that end inside a sample or get no k-block at all, and padding columns filled with NaN.

Bounds (U = 2^-24, the fp32 unit roundoff):
- split-bf16 GEMM results: |got - want| <= 2^-15 * S + tiny elementwise, S = the float64 sum of |a||b| over the same
  contraction, formed from the factors without materialising the generated operand.  Each operand is split into
  bf16 hi + lo with |x - hi - lo| <= 2^-17 |x|; the three products hi*hi + hi*lo + lo*hi drop lo*lo (<= 2^-16 of
  |a||b|) and the residuals, so one product is off by at most 2^-16 |a||b|; the other half of 2^-15 covers the fp32
  accumulation of these zero-mean sums, as for the plain split-bf16 GEMM (test_abi_dense_gpu.py, DESIGN.md section 5).
  A bias is added in fp32 (U * |pre-activation|), and relu / sigmoid are 1-Lipschitz, so the bound carries through
  them; sigmoid's expf and division add at most 8 U.
- the CIN fold: the bound of dZ propagated through the fold (sum |factor| * 2^-15 * S_dZ) plus depth * U times the
  same sum for the fp32 products, partial sums and red.add of the epilogue.
- results rounded once (the outer product, the factor table and its gradient, row unpadding, the gradient
  expansion, the sum over D in ascending d): bit for bit.
- cin_outer_bwd (fp32, may contract to FMA): depth * 2^-23 * sum |terms|.
"""
import pytest
import torch

pytestmark = pytest.mark.gpu

U = 2.0 ** -24                 # unit roundoff of fp32
SPLIT = 2.0 ** -15             # split-bf16 GEMM, relative to sum |a||b| (DESIGN.md section 5)
TINY = 1e-30                   # absolute floor of the bounds (no result here is near the fp32 underflow)
C3 = dict(B=32768, m=26, D=16)
C4 = dict(B=8192, T=50, E=64, n=80)


def _kern():
    from deepctr_b200 import kernels as K, _lib as L
    return K, L


def _rand(gen, shape, dev, std=1.0, mean=0.0):
    return torch.randn(shape, generator=gen, device=dev, dtype=torch.float32) * std + mean


def _within(got, want, bound, what):
    """Elementwise |got - want| <= bound, every value of got finite."""
    assert bool(torch.isfinite(got).all()), "%s: non-finite values" % what
    ratio = (got.double() - want).abs() / bound
    worst = float(ratio.max())
    assert worst <= 1.0, "%s: error %.3g times the bound at %s" % (
        what, worst, tuple(int(i) for i in torch.nonzero(ratio == ratio.max())[0]))


def _act64(act, v):
    from deepctr_b200 import _lib as L
    return {L.ACT_NONE: lambda t: t, L.ACT_RELU: torch.relu, L.ACT_SIGMOID: torch.sigmoid}[act](v)


def _epilogue_bound(S, pre, act):
    """2^-15 S of the GEMM, one fp32 rounding of the bias add, and the activation's own rounding."""
    from deepctr_b200 import _lib as L
    return SPLIT * S + U * pre.abs() + (8 * U if act == L.ACT_SIGMOID else 0.0) + TINY


# ================================================================================================
# CIN factors: T0 [rows, ld0] (columns >= m are padding), X_k [rows, ldk] (columns >= h are not read)
# ================================================================================================
def _cin_factors(gen, dev, rows, m, h, ldk, layer0, poison, mean=0.0, std=0.5):
    """T0 and X_k with padding columns that hold garbage (random) or NaN: the kernels must ignore both.
    Layer 0 reads X_k = T0 (ldk = ld0, h = m), as ops.cin does."""
    ld0 = 32 if m <= 32 else (m + 63) // 64 * 64
    t0 = _rand(gen, (rows, ld0), dev, std, mean)
    if layer0:
        assert h == m
        xk, ldk = t0, ld0
    else:
        xk = _rand(gen, (rows, ldk), dev, std, mean)
    pad = float("nan") if poison else None
    if pad is not None:
        t0[:, m:] = pad
        if not layer0:
            xk[:, h:] = pad
    return t0, xk, ldk


def _cin_fwd64(t0, xk, m, h, w):
    """Y = Z W with Z[r, i*h + j] = t0[r, i] xk[r, j], and S = |Z| |W|, summed over i without materialising Z."""
    t, x = t0[:, :m].double(), xk[:, :h].double()
    w3 = w.double().view(m, h, -1)
    xa, wa = x.abs(), w3.abs()
    y = torch.zeros((t.shape[0], w3.shape[2]), dtype=torch.float64, device=t.device)
    s = torch.zeros_like(y)
    for i in range(m):
        y.addcmul_(t[:, i:i + 1], x @ w3[i])
        s.addcmul_(t[:, i:i + 1].abs(), xa @ wa[i])
    return y, s


def _cin_wgrad64(t0, xk, m, h, dy):
    """dW[i*h + j, n] = sum_r t0[r, i] xk[r, j] dy[r, n] and its sum of |terms|."""
    t, x, d = t0[:, :m].double(), xk[:, :h].double(), dy.double()
    xa, da = x.abs(), d.abs()
    n = d.shape[1]
    dw = torch.empty((m, h, n), dtype=torch.float64, device=d.device)
    s = torch.empty_like(dw)
    for i in range(m):
        dw[i] = (x * t[:, i:i + 1]).t() @ d
        s[i] = (xa * t[:, i:i + 1].abs()).t() @ da
    return dw.view(m * h, n), s.view(m * h, n)


def _filter_planes_and_w(K, gen, dev, m, h, hp, n, std=0.1, mean=0.0):
    w = _rand(gen, (m * h, n), dev, std, mean)
    return w, K.cin_filter_planes(w, m, h, hp)


# (rows, m, h, ldk, n, layer0) of the forward cases; hp = 32 for h <= 32, else h rounded up to 64
_FWD = [
    pytest.param(524288, 26, 26, 32, 128, True, id="c3-layer0"),
    pytest.param(524288, 26, 64, 128, 128, False, id="c3-layer1"),
    pytest.param(4096 * 4, 26, 26, 32, 128, True, id="D4"),
    pytest.param(256 * 128, 26, 64, 128, 128, False, id="D128"),
    pytest.param(1001 * 4, 7, 7, 32, 64, True, id="m7"),
    pytest.param(1001 * 4, 40, 40, 64, 8, True, id="m40-n8"),
    pytest.param(20000, 26, 100, 128, 128, False, id="hp128"),
    pytest.param(9000, 13, 150, 192, 200, False, id="hp192-n200"),
    pytest.param(4100, 5, 256, 256, 64, False, id="hp256-n64"),
]


def _hp(h):
    return 32 if h <= 32 else (h + 63) // 64 * 64


@pytest.mark.parametrize("bias,act", [(True, "relu"), (False, "none"), (True, "sigmoid")])
@pytest.mark.parametrize("rows,m,h,ldk,n,layer0", _FWD)
def test_cin_gemm_forward_matches_float64(cuda, rows, m, h, ldk, n, layer0, bias, act):
    """b2ctr_cin_gemm mode 0: Y = act(Z W' + b) with Z generated by the producer warps; hp >= 128 walks the
    k-blocks j-block-major and keeps X_k in registers across m k-blocks.  Bit-identical from run to run."""
    K, L = _kern()
    a = {"relu": L.ACT_RELU, "none": L.ACT_NONE, "sigmoid": L.ACT_SIGMOID}[act]
    hp = _hp(h)
    gen = torch.Generator(device=cuda).manual_seed(rows + 7 * m + 11 * h + n)
    t0, xk, ldk = _cin_factors(gen, cuda, rows, m, h, ldk, layer0, poison=False)
    w, wp = _filter_planes_and_w(K, gen, cuda, m, h, hp, n)
    b = _rand(gen, (n,), cuda, 0.5) if bias else None
    got = K.cin_gemm(0, t0, xk, ldk, rows, m, h, hp, n, wp, bias=b, act=a)
    again = K.cin_gemm(0, t0, xk, ldk, rows, m, h, hp, n, wp, bias=b, act=a)
    assert torch.equal(got, again), "cin_gemm forward is not deterministic"
    y, s = _cin_fwd64(t0, xk, m, h, w)
    pre = y + b.double() if bias else y
    _within(got, _act64(a, pre), _epilogue_bound(s, pre, a), "cin_gemm mode 0")


@pytest.mark.parametrize("rows,m,h,ldk,n,layer0", [
    pytest.param(524288, 26, 26, 32, 128, True, id="c3-layer0"),
    pytest.param(9000, 26, 150, 192, 128, False, id="hp192"),
])
def test_cin_gemm_forward_ignores_nan_padding(cuda, rows, m, h, ldk, n, layer0):
    """Columns >= m of T0 and >= h of X_k are NaN: the generator loads X_k in float4 units up to the first multiple of
    4 past h, so only the mask of the last partial 8-column group keeps them out of Z."""
    K, L = _kern()
    hp = _hp(h)
    gen = torch.Generator(device=cuda).manual_seed(5 * rows + h)
    t0, xk, ldk = _cin_factors(gen, cuda, rows, m, h, ldk, layer0, poison=True)
    w, wp = _filter_planes_and_w(K, gen, cuda, m, h, hp, n)
    b = _rand(gen, (n,), cuda, 0.5)
    got = K.cin_gemm(0, t0, xk, ldk, rows, m, h, hp, n, wp, bias=b, act=L.ACT_RELU)
    y, s = _cin_fwd64(t0, xk, m, h, w)
    pre = y + b.double()
    _within(got, torch.relu(pre), _epilogue_bound(s, pre, L.ACT_RELU), "cin_gemm mode 0, NaN padding")
    # the filter gradient generates the same operand transposed
    dy = _rand(gen, (rows, n), cuda)
    dwp = K.cin_gemm(1, t0, xk, ldk, rows, m, h, hp, n, K.split_planes(dy))
    want, s = _cin_wgrad64(t0, xk, m, h, dy)
    _within(K.cin_unpad_rows(dwp, m, h, hp), want, SPLIT * s + TINY, "cin_gemm mode 1, NaN padding")
    assert bool((dwp.view(m, hp, n)[:, h:] == 0).all()), "pad rows of dW' must be zero"


def test_cin_gemm_forward_mean_offset(cuda):
    """Positive factors and filter: no cancellation, |Y| is about S, so the bound is exercised at its full size."""
    K, L = _kern()
    rows, m, h, n = 524288, 26, 64, 128
    hp = _hp(h)
    gen = torch.Generator(device=cuda).manual_seed(17)
    t0, xk, ldk = _cin_factors(gen, cuda, rows, m, h, 128, False, poison=False, mean=1.0, std=0.25)
    w, wp = _filter_planes_and_w(K, gen, cuda, m, h, hp, n, std=0.25, mean=1.0)
    got = K.cin_gemm(0, t0, xk, ldk, rows, m, h, hp, n, wp)
    y, s = _cin_fwd64(t0, xk, m, h, w)
    assert float((y / s).min()) > 0.9                 # the test is what it says
    _within(got, y, _epilogue_bound(s, y, L.ACT_NONE), "cin_gemm mode 0, mean offset")


# (rows, m, h, ldk, n, layer0, split_k); split_k None = ops._split_k(m * hp, n, rows)
@pytest.mark.parametrize("rows,m,h,ldk,n,layer0,split_k", [
    pytest.param(524288, 26, 26, 32, 128, True, 1, id="c3-layer0-split1"),
    pytest.param(524288, 26, 26, 32, 128, True, 18, id="c3-layer0-split18"),
    pytest.param(524288, 26, 64, 128, 128, False, 1, id="c3-layer1-split1"),
    pytest.param(524288, 26, 64, 128, 128, False, 10, id="c3-layer1-split10"),
    pytest.param(4096, 26, 64, 128, 128, False, 74, id="empty-slices"),
    pytest.param(1001 * 4, 7, 7, 32, 8, True, None, id="m7-n8"),
    pytest.param(20000, 26, 100, 128, 200, False, None, id="hp128-n200"),
    pytest.param(9000, 13, 150, 192, 64, False, None, id="hp192"),
])
def test_cin_gemm_filter_gradient_matches_float64(cuda, rows, m, h, ldk, n, layer0, split_k):
    """b2ctr_cin_gemm mode 1: dW' = Z^T dY with Z^T generated; split-K over the rows reduced in slice order.  At
    rows = 4096 and 74 slices the slices are 64 rows long and the last 10 get no k-block.  Pad rows (j >= h) of dW'
    are exactly zero.  Bit-identical from run to run."""
    K, L = _kern()
    from deepctr_b200 import ops
    hp = _hp(h)
    if split_k is None:
        split_k = ops._split_k(m * hp, n, rows)
    if rows == 524288:
        # the production split of ops._cin_fused, whenever the test names it
        assert split_k in (1, ops._split_k(m * hp, n, rows))
    gen = torch.Generator(device=cuda).manual_seed(3 * rows + 5 * h + split_k)
    t0, xk, ldk = _cin_factors(gen, cuda, rows, m, h, ldk, layer0, poison=False)
    dy = _rand(gen, (rows, n), cuda)
    planes = K.split_planes(dy)
    dwp = K.cin_gemm(1, t0, xk, ldk, rows, m, h, hp, n, planes, split_k=split_k)
    again = K.cin_gemm(1, t0, xk, ldk, rows, m, h, hp, n, planes, split_k=split_k)
    assert torch.equal(dwp, again), "cin_gemm filter gradient is not deterministic"
    want, s = _cin_wgrad64(t0, xk, m, h, dy)
    _within(K.cin_unpad_rows(dwp, m, h, hp), want, SPLIT * s + TINY, "cin_gemm mode 1")
    if hp > h:
        assert float(dwp.view(m, hp, n)[:, h:].abs().max()) <= TINY, "pad rows of dW' must be zero"


# ================================================================================================
# CIN fold: dZ = dY W'^T folded onto T0 and X_k inside the GEMM epilogue
# ================================================================================================
@pytest.mark.parametrize("m,h,n,layer0", [
    pytest.param(26, 26, 128, True, id="c3-layer0-hp32"),
    pytest.param(26, 64, 128, False, id="c3-layer1-hp64"),
    pytest.param(26, 100, 128, False, id="hp128"),
])
def test_cin_fold_matches_float64(cuda, m, h, n, layer0):
    """b2ctr_cin_fold at C3 rows: dT0[r, i] += sum_j xk[r, j] dZ[r, i*hp + j] and dXk[r, j] += sum_i t0[r, i] dZ[r,
    i*hp + j], with dZ = dY W'^T never stored.  Layer 0 folds both onto dT0 (dxk is dt0, ldx = ld0), as ops.cin does;
    later layers fold dXk into a separate [rows, h] buffer.  red.add makes the order free: bound only."""
    K, L = _kern()
    rows, hp = 524288, _hp(h)
    gen = torch.Generator(device=cuda).manual_seed(29 + h)
    t0, xk, ldk = _cin_factors(gen, cuda, rows, m, h, 128 if h <= 128 else h, layer0, poison=False)
    ld0 = t0.shape[1]
    w, wp = _filter_planes_and_w(K, gen, cuda, m, h, hp, n)
    dy = _rand(gen, (rows, n), cuda)
    dt0 = torch.zeros((rows, ld0), device=cuda)
    dxk = dt0 if layer0 else torch.zeros((rows, h), device=cuda)
    K.cin_fold(t0, xk, ldk, rows, m, h, hp, n, wp, K.split_planes(dy), dt0, dxk, ld0 if layer0 else h)

    t, x, d = t0[:, :m].double(), xk[:, :h].double(), dy.double()
    w3 = w.double().view(m, h, n)
    da = d.abs()
    want_t0 = torch.empty((rows, m), dtype=torch.float64, device=cuda)
    sum_t0 = torch.empty_like(want_t0)
    want_xk = torch.zeros((rows, h), dtype=torch.float64, device=cuda)
    sum_xk = torch.zeros_like(want_xk)
    for i in range(m):
        g = d @ w3[i].t()                     # dZ[:, i*hp : i*hp + h]
        sg = da @ w3[i].abs().t()             # its sum of |terms|: the GEMM bound is 2^-15 sg
        want_t0[:, i] = (x * g).sum(1)
        sum_t0[:, i] = (x.abs() * sg).sum(1)
        want_xk.addcmul_(t[:, i:i + 1], g)
        sum_xk.addcmul_(t[:, i:i + 1].abs(), sg)
    # fp32 fold: a thread sums hp / 8 pairs of products of one output i, two shuffles and a red.add for dT0; m
    # products across the N tiles and a red.add for dXk; layer 0 adds the two into the same element
    depth = hp // 4 + m + 8
    if layer0:
        want_t0 = want_t0 + want_xk
        sum_t0 = sum_t0 + sum_xk
    _within(dt0[:, :m], want_t0, (SPLIT + depth * U) * sum_t0 + TINY, "cin_fold dT0")
    if layer0:
        assert bool((dt0[:, m:] == 0).all()), "cin_fold wrote into the padding columns of dT0"
    else:
        _within(dxk, want_xk, (SPLIT + depth * U) * sum_xk + TINY, "cin_fold dXk")


# ================================================================================================
# DIN: act([q, k, q - k, q * k] W + b) with the attention input generated by the producer warps
# ================================================================================================
def _att_inputs(gen, dev, B, T, E, windowed, std=0.5):
    """query [B, E] and keys [B, T*E], as windows of wider buffers when `windowed` (the query 16 bytes into its row,
    the key rows of a sample further apart than T*E)."""
    if windowed:
        qbuf = _rand(gen, (B, E + 12), dev, std)
        kbuf = _rand(gen, (B, T * E + 8), dev, std)
        return qbuf[:, 4:4 + E], E + 12, kbuf[:, :T * E], T * E + 8
    return _rand(gen, (B, E), dev, std), E, _rand(gen, (B, T * E), dev, std), T * E


def _att_a64(q, keys, B, T, E):
    qd = q.double()[:, None, :].expand(B, T, E)
    kd = keys.double().reshape(B, T, E)
    return torch.cat([qd, kd, qd - kd, qd * kd], dim=-1).reshape(B * T, 4 * E)


@pytest.mark.parametrize("B,T,E,n,windowed", [
    pytest.param(8192, 50, 64, 80, False, id="c4"),
    pytest.param(8192, 50, 64, 80, True, id="c4-windowed"),
    pytest.param(1000, 7, 8, 8, True, id="E8-T7-n8"),
    pytest.param(300, 7, 128, 200, True, id="E128-n200"),
    pytest.param(3000, 1, 64, 80, True, id="T1"),
    pytest.param(777, 7, 16, 64, False, id="E16-n64"),
])
def test_att_gemm_matches_float64(cuda, B, T, E, n, windowed):
    """b2ctr_att_gemm, both modes.  Mode 0 with sigmoid and bias; mode 1 at ops' split (74 at C4: slices of 5568
    rows that end inside a sample of T = 50) and unsplit.  q - k and q * k are rounded to fp32 before the split,
    2^-24 relative per term, inside the bound.  Bit-identical from run to run."""
    K, L = _kern()
    from deepctr_b200 import ops
    rows = B * T
    gen = torch.Generator(device=cuda).manual_seed(B + 3 * T + 5 * E + n)
    q, ldq, keys, kbs = _att_inputs(gen, cuda, B, T, E, windowed)
    w = _rand(gen, (4 * E, n), cuda, 0.1)
    b = _rand(gen, (n,), cuda, 0.5)
    a64 = _att_a64(q, keys, B, T, E)
    aa = a64.abs()

    wp = K.split_planes(w)
    got = K.att_gemm(0, q, ldq, keys, kbs, B, T, E, n, wp, bias=b, act=L.ACT_SIGMOID)
    assert torch.equal(got, K.att_gemm(0, q, ldq, keys, kbs, B, T, E, n, wp, bias=b, act=L.ACT_SIGMOID))
    pre = a64 @ w.double() + b.double()
    _within(got, torch.sigmoid(pre), _epilogue_bound(aa @ w.double().abs(), pre, L.ACT_SIGMOID), "att_gemm mode 0")

    dy = _rand(gen, (rows, n), cuda)
    dyp = K.split_planes(dy)
    want = a64.t() @ dy.double()
    s = aa.t() @ dy.double().abs()
    split = ops._split_k(4 * E, n, rows)
    if (B, T, E, n) == (8192, 50, 64, 80):
        per_slice = -(-(-(-rows // split)) // 64) * 64          # k_per_split of the kernel: 5568 rows
        assert split == 74 and per_slice % T != 0
    for sk in sorted({1, split}):
        dw = K.att_gemm(1, q, ldq, keys, kbs, B, T, E, n, dyp, split_k=sk)
        assert torch.equal(dw, K.att_gemm(1, q, ldq, keys, kbs, B, T, E, n, dyp, split_k=sk))
        _within(dw, want, SPLIT * s + TINY, "att_gemm mode 1, split_k %d" % sk)


# ================================================================================================
# Padded filter planes and the SIMT helpers
# ================================================================================================
@pytest.mark.parametrize("m,h,n", [(26, 26, 128), (26, 64, 128), (7, 150, 200), (13, 100, 8), (3, 256, 64)])
def test_cin_filter_planes_match_split_planes(cuda, m, h, n):
    """b2ctr_cin_filter_planes(W) == b2ctr_split_planes(W') for W' = W with zero rows h <= j < hp in every block i,
    byte for byte except the trailing 256 alignment bytes."""
    K, L = _kern()
    hp = _hp(h)
    gen = torch.Generator(device=cuda).manual_seed(m * h + n)
    w = _rand(gen, (m * h, n), cuda)
    wpad = torch.zeros((m, hp, n), device=cuda)
    wpad[:, :h] = w.view(m, h, n)
    got = K.cin_filter_planes(w, m, h, hp)
    want = K.split_planes(wpad.view(m * hp, n))
    assert got.numel() == want.numel()
    assert torch.equal(got[:-256], want[:-256])


def _rows_of(x, B, m, D):
    """X(b, i, d) of a [B, m*D] buffer as [(b, d), i]"""
    return x.reshape(B, m, D).permute(0, 2, 1).reshape(B * D, m)


_SHAPES = [pytest.param(32768, 26, 16, id="c3"), pytest.param(1001, 7, 4, id="odd")]


@pytest.mark.parametrize("B,m,D", _SHAPES)
def test_cin_t0_and_its_gradient(cuda, B, m, D):
    """cin_t0: T0[(b, d), i] = X0(b, i, d), zero in the padding columns; cin_t0_bwd writes or adds it back into a
    [B, m, D] window.  Both round once (or not at all): bit for bit."""
    K, L = _kern()
    gen = torch.Generator(device=cuda).manual_seed(B + m)
    ld0 = 32 if m <= 32 else (m + 63) // 64 * 64
    xbuf = _rand(gen, (B, m * D + 8), cuda)                 # the field embeddings as a window of a wider row
    x = xbuf[:, :m * D]
    t0 = K.cin_t0(x, (m * D + 8, D, 1), B, m, D, ld0)
    want = torch.zeros((B * D, ld0), device=cuda)
    want[:, :m] = _rows_of(x, B, m, D)
    assert torch.equal(t0, want)

    dt0 = _rand(gen, (B * D, ld0), cuda)
    for acc in (False, True):
        dbuf = _rand(gen, (B, m * D + 4), cuda)
        before = dbuf.clone()
        K.cin_t0_bwd(dt0, ld0, dbuf, (m * D + 4, D, 1), acc, B, m, D)
        back = dt0[:, :m].reshape(B, D, m).permute(0, 2, 1).reshape(B, m * D)
        assert torch.equal(dbuf[:, :m * D], before[:, :m * D] + back if acc else back)
        assert torch.equal(dbuf[:, m * D:], before[:, m * D:])


@pytest.mark.parametrize("m,h,n", [(26, 26, 128), (26, 64, 128), (7, 150, 200)])
def test_cin_unpad_rows(cuda, m, h, n):
    K, L = _kern()
    hp = _hp(h)
    src = _rand(torch.Generator(device=cuda).manual_seed(h), (m * hp, n), cuda)
    assert torch.equal(K.cin_unpad_rows(src, m, h, hp), src.view(m, hp, n)[:, :h].reshape(m * h, n))


@pytest.mark.parametrize("B,m,D", _SHAPES)
def test_cin_sum_d_and_expand_grad(cuda, B, m, D):
    """cin_sum_d: out[b, out_col + c] = sum over d of y[(b, d), col0 + c], added in ascending d from 0 (bit for bit
    with that fp32 sum); the other columns of out stay.  cin_expand_grad: the transpose, plus the hidden-map gradient
    of the next layer over its first hcols columns (one fp32 add)."""
    K, L = _kern()
    gen = torch.Generator(device=cuda).manual_seed(3 * B + D)
    rows, size, col0, ncols, ldo, out_col = B * D, 128, 64, 64, 200, 37
    y = _rand(gen, (rows, size), cuda)
    out = _rand(gen, (B, ldo), cuda)
    before = out.clone()
    K.cin_sum_d(y, size, col0, ncols, D, out, ldo, out_col, 0, B)
    y3 = y.view(B, D, size)
    s = torch.zeros((B, ncols), device=cuda)
    for d in range(D):
        s = s + y3[:, d, col0:col0 + ncols]
    assert torch.equal(out[:, out_col:out_col + ncols], s)
    keep = torch.ones(ldo, dtype=torch.bool, device=cuda)
    keep[out_col:out_col + ncols] = False
    assert torch.equal(out[:, keep], before[:, keep])

    hcols = 64
    dh = _rand(gen, (rows, hcols + 4), cuda)
    for with_dh in (False, True):
        dy = torch.empty((rows, size), device=cuda)
        K.cin_expand_grad(out, ldo, out_col, col0, ncols, dh if with_dh else None, hcols + 4, hcols if with_dh else 0,
                          dy, size, D, 0, B)
        want = torch.zeros((rows, size), device=cuda)
        want[:, col0:col0 + ncols] = out[:, out_col:out_col + ncols].repeat_interleave(D, dim=0)
        if with_dh:
            want[:, :hcols] = want[:, :hcols] + dh[:, :hcols]
        assert torch.equal(dy, want)


# (B, m, D, h, hp, layer0): layer 0 reads X_k = X0 and folds both factors into the same dx (ops._cin_fused's
# non-fold path: T0 seen through strides, hp = 32 > h = 26); later layers read the previous layer's [rows, N] output
@pytest.mark.parametrize("B,m,D,h,hp,layer0", [
    pytest.param(4096, 26, 16, 26, 32, True, id="c3-layer0-hp32"),
    pytest.param(4096, 26, 16, 26, 26, True, id="c3-layer0-dense"),
    pytest.param(4096, 26, 16, 64, 64, False, id="c3-layer1-h64"),
    pytest.param(4096, 26, 16, 40, 64, False, id="h40-hp64"),
    pytest.param(1001, 7, 4, 7, 32, True, id="odd-layer0"),
    pytest.param(1001, 7, 4, 12, 32, False, id="odd-layer1"),
])
def test_cin_outer_fwd_and_bwd(cuda, B, m, D, h, hp, layer0):
    """cin_outer_fwd (one rounded product per element: bit for bit) and cin_outer_bwd over two batch chunks (b0 > 0
    for the second): dX0 (+)= sum_j dZ[i*hp + j] Xk_j, dXk (+)= sum_i dZ[i*hp + j] X0_i; bound depth * 2^-23 *
    sum|terms| with depth = m + h / 32 + 7 (the i loop, the lanes' j loop, the warp sum and the accumulate)."""
    K, L = _kern()
    gen = torch.Generator(device=cuda).manual_seed(B + 13 * h + hp)
    rows, ls = B * D, 2 * h                       # a later layer's input: the first h columns of a [rows, 2h] output
    x = _rand(gen, (B, m * D), cuda)
    v0 = (m * D, D, 1)
    x0r = _rows_of(x, B, m, D)
    if layer0:
        src, vk, xkr = x, v0, x0r
    else:
        src = _rand(gen, (rows, ls), cuda)
        vk, xkr = (D * ls, 1, ls), src[:, :h]

    c = B // 3                                    # two chunks, the second starting at sample c
    for b0, nb in ((0, c), (c, B - c)):
        z = torch.empty((nb * D, m * h), device=cuda)
        K.cin_outer_fwd(x, v0, src, vk, z, b0, nb, m, h, D)
        r = slice(b0 * D, (b0 + nb) * D)
        assert torch.equal(z, (x0r[r, :, None] * xkr[r, None, :]).reshape(nb * D, m * h))

    dz = _rand(gen, (rows, m * hp), cuda)
    dx = _rand(gen, (B, m * D), cuda)             # accumulated into (acc0)
    dx_init = dx.clone()
    dh = None if layer0 else _rand(gen, (rows, h), cuda)     # overwritten (acck = False)
    for b0, nb in ((0, c), (c, B - c)):
        dzc = dz[b0 * D:(b0 + nb) * D]
        if layer0:
            K.cin_outer_bwd(dzc, x, v0, src, vk, dx, v0, True, dx, v0, True, b0, nb, m, h, D, hp)
        else:
            K.cin_outer_bwd(dzc, x, v0, src, vk, dx, v0, True, dh, (D * h, 1, h), False, b0, nb, m, h, D, hp)

    g = dz.double().view(rows, m, hp)[:, :, :h]
    xd, kd = x0r.double(), xkr.double()
    d0 = torch.einsum("rij,rj->ri", g, kd)
    s0 = torch.einsum("rij,rj->ri", g.abs(), kd.abs())
    dk = torch.einsum("rij,ri->rj", g, xd)
    sk = torch.einsum("rij,ri->rj", g.abs(), xd.abs())
    depth = m + h // 32 + 7

    def back(t):                                  # [(b, d), i] -> [B, m*D]
        return t.reshape(B, D, -1).permute(0, 2, 1).reshape(B, -1)
    init = dx_init.double()
    if layer0:
        _within(dx, init + back(d0 + dk), depth * 2 * U * (init.abs() + back(s0 + sk)) + TINY, "cin_outer_bwd dx")
    else:
        _within(dx, init + back(d0), depth * 2 * U * (init.abs() + back(s0)) + TINY, "cin_outer_bwd dx0")
        _within(dh, dk, depth * 2 * U * sk + TINY, "cin_outer_bwd dxk")


# ================================================================================================
# Rejections: argument errors raised before any launch
# ================================================================================================
@pytest.mark.parametrize("case", ["cin-hp96", "cin-hp-lt-h", "cin-h-not-4-unpadded", "cin-xk-misaligned",
                                  "fold-hp192", "att-E12", "att-ldq"])
def test_generated_gemms_reject_unsupported_arguments(cuda, case):
    K, L = _kern()
    rows, m, n = 256, 4, 8
    gen = torch.Generator(device=cuda).manual_seed(1)
    t0 = _rand(gen, (rows, 32), cuda)
    xk = _rand(gen, (rows, 256), cuda)
    dy = _rand(gen, (rows, n), cuda)
    dyp = K.split_planes(dy)
    if case.startswith("att"):
        E = 12 if case == "att-E12" else 8
        ldq = E if case == "att-E12" else 10
        q = _rand(gen, (rows, ldq), cuda)
        keys = _rand(gen, (rows, 2 * E), cuda)
        wp = K.split_planes(_rand(gen, (4 * E, n), cuda))
        n0 = L.launch_count()
        with pytest.raises(ValueError):
            K.att_gemm(0, q, ldq, keys, 2 * E, rows, 2, E, n, wp)
        with pytest.raises(ValueError):
            K.att_gemm(1, q, ldq, keys, 2 * E, rows, 2, E, n, dyp)
        assert L.launch_count() == n0
        return
    h, hp, ldk, x = {"cin-hp96": (64, 96, 96, xk), "cin-hp-lt-h": (64, 32, 64, xk),
                     "cin-h-not-4-unpadded": (26, 32, 28, xk), "cin-xk-misaligned": (32, 32, 32, xk.view(-1)[1:]),
                     "fold-hp192": (150, 192, 192, xk)}[case]
    w = _rand(gen, (m * h, n), cuda)
    wp = K.cin_filter_planes(w, m, h, max(hp, h))
    n0 = L.launch_count()
    if case == "fold-hp192":
        dt0, dh = torch.zeros((rows, 32), device=cuda), torch.zeros((rows, h), device=cuda)
        with pytest.raises(ValueError):
            K.cin_fold(t0, x, ldk, rows, m, h, hp, n, wp, dyp, dt0, dh, h)
    else:
        with pytest.raises(ValueError):
            K.cin_gemm(0, t0, x, ldk, rows, m, h, hp, n, wp)
        with pytest.raises(ValueError):
            K.cin_gemm(1, t0, x, ldk, rows, m, h, hp, n, dyp)
    assert L.launch_count() == n0


# ================================================================================================
# Op level: ops.cin / ops.din_att_first forward and backward on the engine tape against float64 autograd
# ================================================================================================
# With a linear activation every output and gradient is a polynomial in the inputs, weights and upstream
# gradient.  Running the same float64 restatement on |x|, |W|, |b| and |dY| (q - k becoming |q| + |k|) gives M, the
# sum of |terms| of each output and gradient element.  Every split-bf16 GEMM on a path contributes at most 2^-15 of
# the M of its own result, and an error of an earlier stage enters later ones with the weights of M, so a value
# reached through c GEMM stages is within c * 2^-15 * M.  A CIN layer has one GEMM in the forward and two in the
# backward (dZ, then the fold or the filter gradient), and the backward reads the forward's activations: c = 3L for
# L layers.  The fp32 sums on the paths (bias column sums over 2^19 rows in 256-row blocks and their reduction,
# cin_sum_d over D, the fold's and cin_outer_bwd's chains, the attention input's sum over T) are shorter than 4096
# additions.  An elementwise bound holds for every element; a composition error (a missing chunk, a layer read in
# the wrong order, dT0 not accumulated over layers) is a relative error of order one.
def _cin64(x, ws, bs, layer_size, split_half, act):
    """layers/interaction.py's CIN in float64 on [B, m, D]: Z[(b, d), i*h + j] = X0(b, i, d) X_k(b, j, d)."""
    B, m, D = x.shape
    x0 = x.permute(0, 2, 1).reshape(B * D, m)
    hidden, outs = x0, []
    for i, size in enumerate(layer_size):
        h = hidden.shape[1]
        z = (x0[:, :, None] * hidden[:, None, :]).reshape(B * D, m * h)
        y = act(z @ ws[i] + bs[i])
        if split_half and i != len(layer_size) - 1:
            hidden, direct = y[:, :size // 2], y[:, size // 2:]
        else:
            hidden, direct = y, y
        outs.append(direct.reshape(B, D, -1).sum(1))
    return torch.cat(outs, dim=1)


def _cin64_grads(x, ws, bs, gy, layer_size, split_half, act, chunk=2048):
    """Output and gradients of _cin64, a batch chunk at a time (the CIN is per sample)."""
    ws = [w.double().detach().requires_grad_() for w in ws]
    bs = [b.double().detach().requires_grad_() for b in bs]
    out, dx = [], []
    for b0 in range(0, x.shape[0], chunk):
        xc = x[b0:b0 + chunk].double().detach().requires_grad_()
        y = _cin64(xc, ws, bs, layer_size, split_half, act)
        (y * gy[b0:b0 + chunk].double()).sum().backward()
        out.append(y.detach())
        dx.append(xc.grad)
    return torch.cat(out), torch.cat(dx), [w.grad for w in ws], [b.grad for b in bs]


def _run_cin_op(x, ws, bs, gy, layer_size, split_half, act):
    from deepctr_b200 import engine as E, ops
    xv = E.Var(x.clone(), requires_grad=True)
    wv = [E.Var(w.clone(), requires_grad=True) for w in ws]
    bv = [E.Var(b.clone(), requires_grad=True) for b in bs]
    tape = E.Tape()
    with E.recording(tape):
        y = ops.cin(xv, wv, bv, layer_size, act, split_half)
    out = E.contiguous(y).clone()
    y.requires_grad = True
    E.add_grad(y, gy)
    tape.backward()
    return out, xv.grad.reshape(x.shape), [v.grad.reshape(w.shape) for v, w in zip(wv, ws)], [v.grad for v in bv]


def _cin_case(cuda, B, m, D, layer_size, split_half, seed):
    gen = torch.Generator(device=cuda).manual_seed(seed)
    hs = [m] + [s // 2 if split_half else s for s in layer_size]
    x = _rand(gen, (B, m, D), cuda, 0.5)
    ws = [_rand(gen, (m * hs[i], s), cuda, 0.1) for i, s in enumerate(layer_size)]
    bs = [_rand(gen, (s,), cuda, 0.1) for s in layer_size]
    cols = sum(s // 2 if (split_half and i != len(layer_size) - 1) else s for i, s in enumerate(layer_size))
    gy = _rand(gen, (B, cols), cuda)
    return x, ws, bs, gy


def _check_cin_op(got, x, ws, bs, gy, layer_size, split_half, stage_err, what, dw_err=0.0):
    """got = (out, dx, dW, db) of the engine; elementwise against _cin64 with the bound (stage_err + 4096 U) M, and
    dw_err M more for the filter gradients."""
    lin = lambda t: t  # noqa: E731
    want = _cin64_grads(x, ws, bs, gy, layer_size, split_half, lin)
    mag = _cin64_grads(x.abs(), [w.abs() for w in ws], [b.abs() for b in bs], gy.abs(), layer_size, split_half, lin)
    rel = stage_err + 4096 * U
    _within(got[0], want[0], rel * mag[0] + TINY, what + " out")
    _within(got[1], want[1], rel * mag[1] + TINY, what + " dx")
    for i in range(len(layer_size)):
        _within(got[2][i], want[2][i], (rel + dw_err) * mag[2][i] + TINY, what + " dW%d" % i)
        _within(got[3][i], want[3][i], rel * mag[3][i] + TINY, what + " db%d" % i)


@pytest.mark.parametrize("fold", [True, False])
def test_ops_cin_c3_matches_float64(cuda, fold):
    """ops.cin at the C3 shape (B = 32768, 26 fields of 16, layer_size = (128, 128), split_half): the generated
    forward GEMMs, dT0 accumulated over both layers and folded back by cin_t0_bwd (CIN_FOLD) or dZ in row chunks and
    cin_outer_bwd (hp = 32 != h = 26 at layer 0)."""
    from deepctr_b200 import ops
    B, m, D, layer_size = C3["B"], C3["m"], C3["D"], (128, 128)
    x, ws, bs, gy = _cin_case(cuda, B, m, D, layer_size, True, 41)
    assert ops.cin_fusable(x, layer_size, True)
    old = ops.CIN_FOLD, ops.CIN_DZ_CHUNK_BYTES
    ops.CIN_FOLD = fold
    ops.CIN_DZ_CHUNK_BYTES = 128 << 20            # non-fold: dZ of layer 1 in 16 row chunks
    try:
        got = _run_cin_op(x, ws, bs, gy, layer_size, True, "linear")
    finally:
        ops.CIN_FOLD, ops.CIN_DZ_CHUNK_BYTES = old
    _check_cin_op(got, x, ws, bs, gy, layer_size, True, 3 * len(layer_size) * SPLIT, "ops.cin C3")


def test_ops_cin_hp192_non_fold(cuda):
    """layer_size = (384, 128), split_half: layer 1 has h = hp = 192 (the forward's three j-blocks per i), so the fold
    is off and dZ = dY W'^T goes through b2ctr_gemm with the padded filter planes, in three row chunks, then
    cin_outer_bwd with hp = 32 != h = 26 at layer 0."""
    from deepctr_b200 import ops
    B, m, D, layer_size = 4096, 26, 16, (384, 128)
    x, ws, bs, gy = _cin_case(cuda, B, m, D, layer_size, True, 43)
    assert ops.cin_fusable(x, layer_size, True) and ops.CIN_FOLD
    got = _run_cin_op(x, ws, bs, gy, layer_size, True, "linear")
    _check_cin_op(got, x, ws, bs, gy, layer_size, True, 3 * len(layer_size) * SPLIT, "ops.cin hp192")


def test_ops_cin_fp32_path(cuda):
    """set_gemm_precision('fp32'): ops._cin with the outer product materialised per batch chunk (18 chunks of 236
    samples at 26 x 16, hidden width 64) and the exact-fp32 GEMM.  Its sums are fp32 sums in any order: k * U
    relative to M per stage for a contraction of length k, k = m * h <= 1664 for the forward and the data gradient,
    and B * D more for the filter gradient accumulated over the chunks."""
    from deepctr_b200 import ops
    B, m, D, layer_size = 4096, 26, 16, (128, 128)
    x, ws, bs, gy = _cin_case(cuda, B, m, D, layer_size, True, 47)
    ops.set_gemm_precision("fp32")
    try:
        assert not ops.cin_fusable(x, layer_size, True)
        got = _run_cin_op(x, ws, bs, gy, layer_size, True, "linear")
    finally:
        ops.set_gemm_precision("bf16x3")
    _check_cin_op(got, x, ws, bs, gy, layer_size, True, 3 * len(layer_size) * m * 64 * U, "ops._cin fp32",
                  dw_err=B * D * U)


def test_ops_cin_c3_sigmoid_normwise(cuda):
    """The same op with sigmoid: bias_act_bwd then writes dZ's operand planes itself (the fused path at 2^19 x 128).
    A sigmoid network has no majorant of the same form (sigmoid(z) is about 1/2 where z is small), so this case is
    compared normwise: max |got - want| <= 2^-12 max |want| per tensor, eight times one GEMM's 2^-15 for the six
    chained GEMM stages of two layers."""
    from deepctr_b200 import ops
    B, m, D, layer_size = C3["B"], C3["m"], C3["D"], (128, 128)
    x, ws, bs, gy = _cin_case(cuda, B, m, D, layer_size, True, 53)
    got = _run_cin_op(x, ws, bs, gy, layer_size, True, "sigmoid")
    want = _cin64_grads(x, ws, bs, gy, layer_size, True, torch.sigmoid)
    pairs = [("out", got[0], want[0]), ("dx", got[1], want[1])]
    pairs += [("dW%d" % i, got[2][i], want[2][i]) for i in range(2)] + [("db%d" % i, got[3][i], want[3][i])
                                                                        for i in range(2)]
    for name, g, w in pairs:
        assert bool(torch.isfinite(g).all()), name
        err = float((g.double() - w).abs().max()) / float(w.abs().max())
        assert err <= 2.0 ** -12, "ops.cin sigmoid %s: normwise error %.3g" % (name, err)


def test_ops_din_att_first_c4_matches_float64(cuda):
    """ops.din_att_first at the C4 shape with bias: the generated forward, dW through the generated transpose split 74
    ways, dA = dZ W^T from the caller planes of dZ and W, folded back onto q and k.  Elementwise, as for the CIN:
    one GEMM stage per value."""
    from deepctr_b200 import engine as E, ops
    B, T, Ed, n = C4["B"], C4["T"], C4["E"], C4["n"]
    gen = torch.Generator(device=cuda).manual_seed(59)
    q = _rand(gen, (B, 1, Ed), cuda, 0.5)
    k = _rand(gen, (B, T, Ed), cuda, 0.5)
    w = _rand(gen, (4 * Ed, n), cuda, 0.1)
    b = _rand(gen, (n,), cuda, 0.1)
    gy = _rand(gen, (B, T, n), cuda)
    vs = [E.Var(t.clone(), requires_grad=True) for t in (q, k, w, b)]
    assert ops.din_att_fusable(vs[0], vs[1], n)
    tape = E.Tape()
    with E.recording(tape):
        y = ops.din_att_first(vs[0], vs[1], vs[2], vs[3], "linear")
    out = E.contiguous(y).clone()
    y.requires_grad = True
    E.add_grad(y, gy)
    tape.backward()

    def ref(q, k, w, b, gy, absmodel):
        ts = [t.double().detach().requires_grad_() for t in (q, k, w, b)]
        qq = ts[0].expand(B, T, Ed)
        a = torch.cat([qq, ts[1], qq + ts[1] if absmodel else qq - ts[1], qq * ts[1]], dim=-1)
        o = a @ ts[2] + ts[3]
        (o * gy.double()).sum().backward()
        return [o.detach()] + [t.grad for t in ts]
    want = ref(q, k, w, b, gy, False)
    mag = ref(q.abs(), k.abs(), w.abs(), b.abs(), gy.abs(), True)
    rel = SPLIT + 4096 * U
    for name, g, wv, mv in zip(("out", "dq", "dk", "dW", "db"), [out] + [v.grad.reshape(v.shape) for v in vs],
                               want, mag):
        _within(g.reshape(wv.shape), wv, rel * mv + TINY, "ops.din_att_first " + name)
