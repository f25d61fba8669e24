"""GPU: the dense tower between the embedding buffer and the loss, against float64 at production shapes.

Covered: the exact-fp32 GEMM (tile kernels in every majorness, both split-K reductions, the skinny-N / skinny-TN /
skinny-K kernels), the split-bf16 GEMM as ops.dense calls it, split_planes, bias_act_bwd (both kernels and the fused
operand planes), the prediction head and loss, the dense optimizers, the unfused FM, the copy / sum plumbing, and
one composed 845 -> 256 -> 128 -> 64 -> 1 tower through ops.dense in both GEMM precisions.

Two kinds of check:
- exact-valued operands: integers times a power of two, chosen so that every partial sum of every reduction stays
  below 2^24 grid units.  Every fp32 sum is then exact whatever its order, so the kernel must equal the float64
  result bit for bit; a dropped or doubled row, k-slice, tile or CTA partial cannot hide in a tolerance.  Each such
  test asserts its own precondition (the sum of |terms| of every output below 2^24 units).
- random operands with a derived bound: an fp32 sum of k terms is within (k + c) * 2^-24 * sum|terms| of the exact
  one; it goes through an activation scaled by the activation's Lipschitz constant (1 for relu / tanh, 1/4 for
  sigmoid), plus a few ulps of the result for expf / tanhf.  The split-bf16 product drops only the lo * lo term,
  at most 2^-16 |a||b| per product, and the bound used is 2^-15 sum |a||b| plus the fp32 accumulation term.

The float64 references run on the device (row-chunked for the largest operands).
"""
import zlib

import numpy as np
import pytest
import torch

from conftest import gemm_precision  # noqa: F401  (the composed tower runs in both GEMM precisions)

pytestmark = pytest.mark.gpu

U = 2.0 ** -24          # fp32 unit roundoff
LIMIT = 2.0 ** 24       # grid units below which every fp32 partial sum is exact
CHUNK = 1 << 16         # rows per float64 reference chunk


def _mods():
    from deepctr_b200 import _lib as L, kernels as K, ops
    return L, K, ops


@pytest.fixture
def gen(cuda, request):
    """device generator seeded from the test id: every parameter set draws its own, reproducible data"""
    g = torch.Generator(device=cuda)
    g.manual_seed(zlib.crc32(request.node.name.encode()))
    return g


def _ints(gen, shape, lo, hi, scale):
    """integers in [lo, hi] times ``scale`` (a power of two), fp32 on the device"""
    return torch.randint(lo, hi + 1, shape, generator=gen, device=gen.device).float() * scale


def _randn(gen, shape, scale=1.0):
    return torch.randn(shape, generator=gen, device=gen.device) * scale


def _mm64(a, b):
    """float64 a @ b on the device, in row chunks of a"""
    b = b.double()
    out = torch.empty((a.shape[0], b.shape[1]), dtype=torch.float64, device=a.device)
    for r in range(0, a.shape[0], CHUNK):
        out[r:r + CHUNK] = a[r:r + CHUNK].double() @ b
    return out


def _atb64(a, b):
    """float64 a^T @ b on the device for tall a, b (a reduction over the rows), in row chunks"""
    out = torch.zeros((a.shape[1], b.shape[1]), dtype=torch.float64, device=a.device)
    for r in range(0, a.shape[0], CHUNK):
        out += a[r:r + CHUNK].double().t() @ b[r:r + CHUNK].double()
    return out


def _op(t, trans):
    return t.t() if trans else t


def _act64(v, act):
    L, _, _ = _mods()
    if act == L.ACT_RELU:
        return torch.relu(v)
    if act == L.ACT_SIGMOID:
        return torch.sigmoid(v)
    if act == L.ACT_TANH:
        return torch.tanh(v)
    return v


def _lip(act):
    L, _, _ = _mods()
    return 0.25 if act == L.ACT_SIGMOID else 1.0


def _exact_ok(absum, unit):
    """precondition of an exact-valued check: sum|terms| of every output below 2^24 units of the grid"""
    assert float(absum.max()) < LIMIT * unit, (float(absum.max()) / unit, LIMIT)


def _assert_within(got, ref, bound, what=""):
    err = (got.double() - ref).abs()
    assert bool(torch.isfinite(got).all()), what + ": non-finite output"
    ok = err <= bound
    if not bool(ok.all()):
        i = int((err - bound).argmax())
        raise AssertionError("%s: %d elements out of bound; worst |err| %.3e vs bound %.3e (flat index %d)" % (
            what, int((~ok).sum()), float(err.flatten()[i]), float(bound.flatten()[i]), i))


def _assert_equal(got, ref, what=""):
    """bit-for-bit: ref is float64 and exactly representable in fp32"""
    want = ref.float()
    assert bool((want.double() == ref).all()), what + ": reference not representable in fp32 (test bug)"
    if not torch.equal(got, want):
        d = (got.double() - ref).abs()
        raise AssertionError("%s: %d elements differ, max |diff| %.3e" % (what, int((d > 0).sum()),
                                                                          float(d.max())))


def _padded(gen, rows, cols, ld, fill, lo, hi, scale):
    """[rows, cols] exact-valued window of a [rows, ld] buffer whose other columns hold ``fill``"""
    buf = torch.full((rows, ld), fill, device=gen.device)
    buf[:, :cols] = _ints(gen, (rows, cols), lo, hi, scale)
    return buf, buf[:, :cols]


# ---- exact-fp32 GEMM: the tower shapes -------------------------------------------------------------------------
# (B, k, n): C2 = DeepFM at B = 65536, 845 -> 256 -> 128 -> 64 -> 1; C3 = xDeepFM's DNN at B = 32768 (429 -> 256);
# C4 = DIN's attention MLP over 409600 (sample, behaviour) rows, 256 -> 80 -> 40 -> 1
TOWER = [(65536, 845, 256), (65536, 256, 128), (65536, 128, 64), (65536, 64, 1), (32768, 429, 256),
         (409600, 256, 80), (409600, 80, 40), (409600, 40, 1)]
TOWER_IDS = ["%dx%d-%d" % s for s in TOWER]


@pytest.mark.parametrize("B,k,n", TOWER, ids=TOWER_IDS)
def test_gemm_fp32_tower_exact(cuda, gen, B, k, n):
    """forward (bias + relu), dgrad into the K-padded [B, ld] buffer (sentinel in the pad columns) and the split-K
    wgrad at ops._split_k's slice count, each equal to float64 on exact-valued operands.  The forward operand's pad
    columns hold NaN: a kernel that reads past k produces NaN."""
    L, K, ops = _mods()
    ld = (k + 3) // 4 * 4
    amp = 8 if B * 64 < LIMIT else 4                 # |terms| <= amp^2 units of 2^-8 on a k = B reduction
    xbuf, x = _padded(gen, B, k, ld, float("nan"), -amp, amp, 2.0 ** -4)
    w = _ints(gen, (k, n), -8, 8, 2.0 ** -4)
    bias = _ints(gen, (n,), -64, 64, 2.0 ** -8)
    y = K.gemm(x, w, bias=bias, act=L.ACT_RELU, m=B, n=n, k=k)
    _exact_ok(_mm64(x.abs(), w.abs()) + bias.abs().double(), 2.0 ** -8)
    _assert_equal(y, torch.relu(_mm64(x, w) + bias.double()), "forward")
    # dgrad: dX = dZ W^T written into the window of a K-padded buffer; the pad columns must keep their sentinel
    dz = _ints(gen, (B, n), -amp, amp, 2.0 ** -4)
    dxbuf = torch.full((B, ld), -3.25, device=cuda)
    K.gemm(dz, w, c=dxbuf[:, :k], trans_b=True, m=B, n=k, k=n)
    _assert_equal(dxbuf[:, :k], _mm64(dz, w.t()), "dgrad")
    assert bool((dxbuf[:, k:] == -3.25).all()), "dgrad wrote outside its window"
    # wgrad: dW = X^T dZ, K = B split as ops.dense splits it
    sk = ops._split_k(k, n, B)
    dw = K.gemm(x, dz, trans_a=True, split_k=sk, m=k, n=n, k=B)
    _exact_ok(_atb64(x.abs(), dz.abs()), 2.0 ** -8)
    _assert_equal(dw, _atb64(x, dz), "wgrad (split_k=%d)" % sk)


# ---- exact-fp32 GEMM: every tile width in every majorness ------------------------------------------------------
@pytest.mark.parametrize("n", [30, 60, 250], ids=["bn32", "bn64", "bn128"])
@pytest.mark.parametrize("ta,tb", [(False, False), (False, True), (True, False), (True, True)])
@pytest.mark.parametrize("sk", [1, 3])
def test_gemm_fp32_tiles_all_layouts_exact(cuda, gen, n, ta, tb, sk):
    """2000 x n x 300 (16 row tiles, 1 or 2 column tiles) from [m, k] / [k, m] A and [k, n] / [n, k] B: bias + relu
    into a fresh C, then alpha = 0.5 accumulated into a window of a wider C whose outside columns must stay put"""
    L, K, _ = _mods()
    m, k = 2000, 300
    a = _ints(gen, (k, m) if ta else (m, k), -8, 8, 2.0 ** -4)
    b = _ints(gen, (n, k) if tb else (k, n), -8, 8, 2.0 ** -4)
    bias = _ints(gen, (n,), -64, 64, 2.0 ** -8)
    ref = _mm64(_op(a, ta), _op(b, tb))
    _exact_ok(_mm64(_op(a, ta).abs(), _op(b, tb).abs()), 2.0 ** -8)
    got = K.gemm(a, b, bias=bias, act=L.ACT_RELU, trans_a=ta, trans_b=tb, split_k=sk, m=m, n=n, k=k)
    _assert_equal(got, torch.relu(ref + bias.double()), "bias + relu")
    cbuf = torch.full((m, n + 5), 11.5, device=cuda)
    c0 = _ints(gen, (m, n), -64, 64, 2.0 ** -8)
    cbuf[:, 2:n + 2] = c0
    K.gemm(a, b, c=cbuf[:, 2:n + 2], trans_a=ta, trans_b=tb, accumulate=True, alpha=0.5, split_k=sk, m=m, n=n, k=k)
    _assert_equal(cbuf[:, 2:n + 2], c0.double() + 0.5 * ref, "alpha + accumulate")
    assert bool((cbuf[:, :2] == 11.5).all()) and bool((cbuf[:, n + 2:] == 11.5).all()), "wrote outside C's window"


@pytest.mark.parametrize("act", ["none", "relu", "sigmoid", "tanh"])
@pytest.mark.parametrize("m,n,k,ta,sk", [(1000, 200, 845, False, 1), (845, 256, 8192, True, 4), (4096, 40, 80, False, 1)])
def test_gemm_fp32_activations_random_bound(cuda, gen, act, m, n, k, ta, sk):
    """random operands, alpha = 0.75 and bias, each activation (in the split-K reduction when sk > 1)"""
    L, K, _ = _mods()
    a_code = L.ACT_BY_NAME[None if act == "none" else act]
    a = _randn(gen, (k, m) if ta else (m, k))
    b = _randn(gen, (k, n), 0.1)
    bias = _randn(gen, (n,))
    got = K.gemm(a, b, bias=bias, act=a_code, alpha=0.75, trans_a=ta, split_k=sk, m=m, n=n, k=k)
    A = _op(a, ta)
    ref = _act64(0.75 * _mm64(A, b) + bias.double(), a_code)
    absum = 0.75 * _mm64(A.abs(), b.abs()) + bias.abs().double()
    bound = _lip(a_code) * (k + sk + 4) * U * absum + 8 * U * ref.abs() + 1e-30
    _assert_within(got, ref, bound, act)


# ---- both split-K reductions -----------------------------------------------------------------------------------
@pytest.mark.parametrize("m,n,k,sk,kind", [
    (64, 64, 65536, 64, "small"),      # m n <= 4096 and >= 16 slices: one warp per output (tile kernel)
    (13, 1, 65536, 256, "small"),      # the dense features' [13, 1] wgrad (16-k-lane skinny-TN kernel)
    (64, 1, 65536, 256, "small"),      # the last projection's [64, 1] wgrad (vec4 skinny-TN kernel)
    (64, 64, 65536, 8, "plain"),       # few slices: one thread per output
    (845, 256, 65536, 18, "plain"),    # the C2 first layer's wgrad
    (96, 48, 65536, 32, "plain"),      # m n > 4096 with many slices
])
@pytest.mark.parametrize("mode", ["accumulate", "bias_relu"])
def test_gemm_fp32_splitk_reductions_exact(cuda, gen, m, n, k, sk, kind, mode):
    """wgrad-shaped GEMMs whose slices meet in splitk_reduce_small_kernel or splitk_reduce_kernel: every slice must
    be added exactly once (equality with float64 on exact-valued operands), epilogue applied after the sum"""
    L, K, _ = _mods()
    ld = m + 4
    a = torch.full((k, ld), float("nan"), device=cuda)
    a[:, :m] = _ints(gen, (k, m), -4, 4, 2.0 ** -4)
    a = a[:, :m]
    b = _ints(gen, (k, n), -4, 4, 2.0 ** -4)
    ref = _atb64(a, b)
    _exact_ok(_atb64(a.abs(), b.abs()), 2.0 ** -8)
    if mode == "accumulate":
        cbuf = torch.full((m, n + 3), -1.5, device=cuda)
        c0 = _ints(gen, (m, n), -64, 64, 2.0 ** -8)
        cbuf[:, :n] = c0
        K.gemm(a, b, c=cbuf[:, :n], trans_a=True, accumulate=True, alpha=0.5, split_k=sk, m=m, n=n, k=k)
        _assert_equal(cbuf[:, :n], c0.double() + 0.5 * ref, kind)
        assert bool((cbuf[:, n:] == -1.5).all())
    else:
        bias = _ints(gen, (n,), -64, 64, 2.0 ** -8)
        got = K.gemm(a, b, bias=bias, act=L.ACT_RELU, trans_a=True, split_k=sk, m=m, n=n, k=k)
        _assert_equal(got, torch.relu(ref + bias.double()), kind)


# ---- skinny kernels --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("k,lda,off,path", [
    (45, 47, 0, "scalar"),           # lda % 4 != 0
    (64, 64, 1, "scalar"),           # rows not 16-byte aligned
    (64, 64, 0, "vec-fast"),         # k <= 4 lanes x 32: one float4 per lane
    (45, 48, 0, "vec-fast-pad"),     # k % 4 != 0: the last float4 reaches into the row's NaN padding
    (17, 20, 0, "vec-fast-pad"),
    (127, 128, 0, "vec-fast-pad"),
    (845, 848, 0, "vec-loop"),       # k > 128: the strided float4 loop
])
@pytest.mark.parametrize("n", [1, 2, 3, 8])
@pytest.mark.parametrize("tb", [False, True])
def test_gemm_fp32_skinny_n_exact(cuda, gen, k, lda, off, path, n, tb):
    """A row-major, N <= 8: the [*, 1] projection's forward.  The A buffer's pad columns hold NaN, which must never
    reach C; alpha + accumulate into a C window and bias + relu, both exact."""
    L, K, _ = _mods()
    m = 65537
    buf = torch.full((m * lda + 4,), float("nan"), device=cuda)
    a = buf[off:off + m * lda].view(m, lda)
    a[:, :k] = _ints(gen, (m, k), -8, 8, 2.0 ** -4)
    a = a[:, :k]
    b = _ints(gen, (n, k) if tb else (k, n), -8, 8, 2.0 ** -4)
    ref = _mm64(a, _op(b, tb))
    bias = _ints(gen, (n,), -64, 64, 2.0 ** -8)
    got = K.gemm(a, b, bias=bias, act=L.ACT_RELU, trans_b=tb, m=m, n=n, k=k)
    _assert_equal(got, torch.relu(ref + bias.double()), path + " bias + relu")
    cbuf = torch.full((m, n + 3), 2.5, device=cuda)
    c0 = _ints(gen, (m, n), -64, 64, 2.0 ** -8)
    cbuf[:, :n] = c0
    K.gemm(a, b, c=cbuf[:, :n], trans_b=tb, accumulate=True, alpha=0.5, m=m, n=n, k=k)
    _assert_equal(cbuf[:, :n], c0.double() + 0.5 * ref, path + " alpha + accumulate")
    assert bool((cbuf[:, n:] == 2.5).all())


@pytest.mark.parametrize("m,n,lda,kernel", [
    (13, 1, 16, "16-k-lane"),        # the dense features' [13, 1] wgrad
    (64, 1, 68, "vec4"),
    (64, 2, 64, "vec4"),
    (128, 1, 129, "scalar"),         # lda % 4 != 0
    (65, 1, 68, "scalar"),           # m % 4 != 0
    (40, 3, 40, "scalar"),           # n in 3..8
    (100, 8, 104, "scalar"),
])
@pytest.mark.parametrize("B", [4097, 65536])
def test_gemm_fp32_skinny_tn_exact(cuda, gen, m, n, lda, kernel, B):
    """A stored [K, M] (trans_a), N <= 8: the skinny wgrads, without and with split-K at ops._split_k's count"""
    L, K, ops = _mods()
    a = torch.full((B, lda), float("nan"), device=cuda)
    a[:, :m] = _ints(gen, (B, m), -4, 4, 2.0 ** -4)
    a = a[:, :m]
    b = _ints(gen, (B, n), -4, 4, 2.0 ** -4)
    ref = _atb64(a, b)
    _exact_ok(_atb64(a.abs(), b.abs()), 2.0 ** -8)
    for sk in sorted({1, ops._split_k(m, n, B)}):
        got = K.gemm(a, b, trans_a=True, split_k=sk, m=m, n=n, k=B)
        _assert_equal(got, ref, "%s split_k=%d" % (kernel, sk))


@pytest.mark.parametrize("n,ldc,off,path", [(64, 64, 0, "float4 C"), (845, 848, 0, "float4 C + tail"),
                                            (845, 847, 0, "scalar C"), (256, 260, 1, "scalar C")])
@pytest.mark.parametrize("k", [1, 5])
def test_gemm_fp32_skinny_k_exact(cuda, gen, n, ldc, off, path, k):
    """A row-major, K <= 8, N >= 16: the [*, 1] projection's dgrad (an outer product) into a strided C window"""
    L, K, _ = _mods()
    m = 65536
    a = _ints(gen, (m, k), -8, 8, 2.0 ** -4)
    b = _ints(gen, (n, k), -8, 8, 2.0 ** -4)      # stored [N, K]: W^T of a [n, k] weight, as ops.dense passes it
    ref = _mm64(a, b.t())
    buf = torch.full((m * ldc + 4,), 6.0, device=cuda)
    cv = buf[off:off + m * ldc].view(m, ldc)
    c0 = _ints(gen, (m, n), -64, 64, 2.0 ** -8)
    cv[:, :n] = c0
    K.gemm(a, b, c=cv[:, :n], trans_b=True, accumulate=True, alpha=0.5, m=m, n=n, k=k)
    _assert_equal(cv[:, :n], c0.double() + 0.5 * ref, path)
    assert bool((cv[:, n:] == 6.0).all()) and bool((buf[:off] == 6.0).all())
    bias = _ints(gen, (n,), -64, 64, 2.0 ** -8)
    got = K.gemm(a, b, bias=bias, act=L.ACT_RELU, trans_b=True, m=m, n=n, k=k)
    _assert_equal(got, torch.relu(ref + bias.double()), path + " bias + relu")


# ---- split-bf16 GEMM (variant 0, what ops.dense calls) ---------------------------------------------------------
# (m, n, k, trans_a, trans_b, split_k): forward, dgrad and wgrad of the C2 / C3 / C4 layers with min(n, k) >= 16
def _bf16_shapes():
    out = []
    for B, k, n in TOWER:
        if min(k, n) < 16:
            continue
        out += [(B, n, k, False, False, 1, "fwd"), (B, k, n, False, True, 1, "dgrad")]
        out.append((k, n, B, True, False, None, "wgrad"))         # split_k: ops._split_k, as ops.dense passes it
    return out


BF16 = _bf16_shapes()


@pytest.mark.parametrize("m,n,k,ta,tb,sk,kind", BF16, ids=["%s-%dx%dx%d" % (s[6], s[0], s[1], s[2]) for s in BF16])
def test_gemm_bf16x3_tower_bound(cuda, gen, m, n, k, ta, tb, sk, kind):
    """random operands against float64: 2^-15 sum|a||b| plus the fp32 accumulation term; the forward with bias and
    each activation"""
    L, K, ops = _mods()
    sk = sk or ops._split_k(m, n, k)
    a = _randn(gen, (k, m) if ta else (m, k))
    b = _randn(gen, (n, k) if tb else (k, n), 0.1)
    A, Bm = _op(a, ta), _op(b, tb)
    prod = _atb64(a, Bm) if ta else _mm64(A, Bm)
    absum = _atb64(a.abs(), Bm.abs()) if ta else _mm64(A.abs(), Bm.abs())
    acts = [L.ACT_NONE, L.ACT_RELU, L.ACT_SIGMOID, L.ACT_TANH] if kind == "fwd" else [L.ACT_NONE]
    bias = _randn(gen, (n,)) if kind == "fwd" else None
    for act in acts:
        got = K.gemm(a, b, bias=bias, act=act, trans_a=ta, trans_b=tb, split_k=sk, precision=L.GEMM_BF16X3,
                     m=m, n=n, k=k)
        pre = prod + (bias.double() if bias is not None else 0.0)
        ref = _act64(pre, act)
        full = absum + (bias.abs().double() if bias is not None else 0.0)
        bound = _lip(act) * (2.0 ** -15 * absum + (k + sk + 8) * U * full) + 8 * U * ref.abs() + 1e-30
        _assert_within(got, ref, bound, "%s act=%d" % (kind, act))


@pytest.mark.parametrize("m,n,k,ta,tb,sk,kind", [s for s in BF16 if s[0] * s[1] * s[2] <= 65536 * 845 * 256
                                                  and max(s[0], s[2]) <= 65536],
                         ids=["%s-%dx%dx%d" % (s[6], s[0], s[1], s[2]) for s in BF16
                              if s[0] * s[1] * s[2] <= 65536 * 845 * 256 and max(s[0], s[2]) <= 65536])
def test_gemm_bf16x3_tower_exact(cuda, gen, m, n, k, ta, tb, sk, kind):
    """A with at most 10 significant bits (hi_A + lo_A = A exactly), B bf16-exact (lo_B = 0): the three-term
    product is A B exactly, so the result must equal float64 - a dropped lo plane or k-block shows.  Whether wgmma's
    fp32 accumulation is exact on such sums is not documented; this test is the evidence that it is."""
    L, K, ops = _mods()
    sk = sk or ops._split_k(m, n, k)
    amp = 1023 if k <= 4096 else 511              # keeps sum|a||b| of every output below 2^24 units at k = 65536
    a = _ints(gen, (k, m) if ta else (m, k), -amp, amp, 2.0 ** -10)
    b = _ints(gen, (n, k) if tb else (k, n), -1, 1, 2.0 ** -3)
    A, Bm = _op(a, ta), _op(b, tb)
    assert float((a.to(torch.bfloat16).float() != a).float().mean()) > 0.2     # lo_A != 0 for many elements
    ref = _atb64(a, Bm) if ta else _mm64(A, Bm)
    _exact_ok(_atb64(a.abs(), Bm.abs()) if ta else _mm64(A.abs(), Bm.abs()), 2.0 ** -13)
    got = K.gemm(a, b, trans_a=ta, trans_b=tb, split_k=sk, precision=L.GEMM_BF16X3, m=m, n=n, k=k)
    _assert_equal(got, ref, kind)


# ---- split_planes ----------------------------------------------------------------------------------------------
def _bf16_rne(x):
    """numpy: bf16 bits (uint16) of fp32 x rounded to nearest, ties to even"""
    b = x.view(np.uint32).astype(np.uint64)
    return ((b + 0x7FFF + ((b >> 16) & 1)) >> 16).astype(np.uint16)


def _planes_ref(x):
    """numpy restatement of b2ctr_split_planes: hi = bf16_rn(x), lo = bf16_rn(x - hi); planes [rows_pad, pitch]
    (rows rounded up to 256, pitch 64 or a multiple of 128), hi plane then lo plane, zero outside [rows, cols)"""
    x = np.ascontiguousarray(x, dtype=np.float32)
    rows, cols = x.shape
    rp = (rows + 255) // 256 * 256
    cp = 64 if cols <= 64 else (cols + 127) // 128 * 128
    hi = _bf16_rne(x)
    hif = (hi.astype(np.uint32) << 16).view(np.float32)
    lo = _bf16_rne((x - hif).astype(np.float32))
    out = np.zeros((2, rp, cp), dtype=np.uint16)
    out[0, :rows, :cols] = hi
    out[1, :rows, :cols] = lo
    return out


def _planes_got(buf, rows, cols):
    rp = (rows + 255) // 256 * 256
    cp = 64 if cols <= 64 else (cols + 127) // 128 * 128
    assert buf.numel() == 2 * rp * cp * 2 + 256, "planes_bytes"
    return buf[:-256].cpu().numpy().view(np.uint16).reshape(2, rp, cp)


def _wide_range(gen, shape):
    """normal values over 2^-40 .. 2^40, with rounding ties (low 16 bits 0x8000, both parities of bit 16), values
    one step either side of a tie, subnormals and signed zeros mixed in"""
    x = _randn(gen, shape) * torch.exp2(torch.randint(-40, 41, shape, generator=gen, device=gen.device).float())
    bits = x.view(torch.int32)
    sel = torch.randint(0, 8, shape, generator=gen, device=gen.device)
    hi16 = bits & ~0xFFFF
    bits = torch.where(sel == 1, hi16 | 0x8000, bits)
    bits = torch.where(sel == 2, hi16 | 0x7FFF, bits)
    bits = torch.where(sel == 3, hi16 | 0x8001, bits)
    bits = torch.where(sel == 4, (bits & -2 ** 31) | (bits & 0x007FFFFF), bits)     # subnormal
    x = bits.view(torch.float32)
    x = torch.where(sel == 5, torch.zeros_like(x) * torch.sign(x), x)                  # +0 / -0
    return x


@pytest.mark.parametrize("rows,cols,ld,off", [
    (1, 1, 1, 0), (1, 1, 5, 3),
    (300, 64, 64, 0),                # pitch 64
    (257, 65, 68, 0),                # pitch 128, strided float4 source
    (1000, 845, 848, 0),             # the C2 input window
    (513, 256, 260, 1),              # 16-byte-misaligned source: scalar loads
    (256, 130, 131, 0),              # ld % 4 != 0: scalar loads
    (4096, 40, 40, 0),
])
def test_split_planes_bytes(cuda, gen, rows, cols, ld, off):
    """b2ctr_split_planes byte for byte against the numpy restatement: hi, lo, pitch, row padding, zero pads"""
    _, K, _ = _mods()
    buf = torch.full((rows * ld + off + 4,), float("nan"), device=cuda)
    src = buf[off:off + rows * ld].view(rows, ld)
    src[:, :cols] = _wide_range(gen, (rows, cols))
    x = src[:, :cols]
    got = _planes_got(K.split_planes(x), rows, cols)
    want = _planes_ref(x.cpu().numpy())
    bad = got != want
    assert not bad.any(), "%d bf16 values differ, first at (plane, row, col) %s" % (int(bad.sum()),
                                                                                   tuple(np.argwhere(bad)[0]))


# ---- bias_act_bwd ----------------------------------------------------------------------------------------------
def _act_out(gen, act, shape):
    """exact-valued activation outputs: relu >= 0 (zeros included), sigmoid in (0, 1), tanh in (-1, 1), on 2^-4"""
    L, _, _ = _mods()
    if act == L.ACT_RELU:
        return torch.relu(_ints(gen, shape, -8, 15, 2.0 ** -4))
    if act == L.ACT_SIGMOID:
        return _ints(gen, shape, 1, 15, 2.0 ** -4)
    return _ints(gen, shape, -15, 15, 2.0 ** -4)


def _grad64(y, act):
    L, _, _ = _mods()
    y = y.double()
    if act == L.ACT_RELU:
        return (y > 0).double()
    if act == L.ACT_SIGMOID:
        return y * (1 - y)
    if act == L.ACT_TANH:
        return 1 - y * y
    return torch.ones_like(y)


@pytest.mark.parametrize("n", [4, 8, 64, 128, 256, 1024, 200, 90])
@pytest.mark.parametrize("m", [1, 127, 129, 65536, 65537])
@pytest.mark.parametrize("vec", [True, False], ids=["vec4", "scalar"])
def test_bias_act_bwd_exact(cuda, gen, n, m, vec):
    """dz = dy act'(y) and dbias = colsum(dz) on exact-valued inputs, every activation, on windows with ld > n
    (ld % 4 == 0 keeps the float4 kernel where n allows it, ld odd forces the scalar one); want_dz=False too"""
    L, K, _ = _mods()
    if vec and not (n % 4 == 0 and 256 % (n // 4) == 0):
        pytest.skip("the float4 kernel needs n / 4 to divide 256")
    ld = n + 4 if vec else n + 3
    for act in (L.ACT_NONE, L.ACT_RELU, L.ACT_SIGMOID, L.ACT_TANH):
        dyb = torch.full((m, ld), float("nan"), device=cuda)
        yb = torch.full((m, ld), float("nan"), device=cuda)
        dyb[:, :n] = _ints(gen, (m, n), -1, 1, 2.0 ** -4)
        yb[:, :n] = _act_out(gen, act, (m, n))
        dy, y = dyb[:, :n], yb[:, :n]
        dz_ref = dy.double() * _grad64(y, act)
        _exact_ok(dz_ref.abs().sum(0), 2.0 ** -12)
        dz, db = K.bias_act_bwd(dy, y, act)
        _assert_equal(dz[:, :n], dz_ref, "dz act=%d" % act)
        _assert_equal(db, dz_ref.sum(0), "dbias act=%d" % act)
        dz2, db2 = K.bias_act_bwd(dy, y, act, want_dz=False)
        assert dz2 is None
        _assert_equal(db2, dz_ref.sum(0), "dbias (want_dz=False) act=%d" % act)


@pytest.mark.parametrize("n", [64, 128, 256, 1024])
@pytest.mark.parametrize("act", ["relu", "sigmoid", "tanh"])
def test_bias_act_bwd_fused_planes(cuda, gen, n, act):
    """random dy, y at m = 65536 (8192 for n = 1024): dz within a few ulps of float64, dbias within its summation bound, and the fused
    bf16 planes equal to the numpy restatement of split_planes(dz), with and without dz written"""
    L, K, _ = _mods()
    m = 65536 if n <= 256 else 8192
    a = L.ACT_BY_NAME[act]
    dy = _randn(gen, (m, n))
    z = _randn(gen, (m, n), 2.0)
    y = {"relu": torch.relu, "sigmoid": torch.sigmoid, "tanh": torch.tanh}[act](z)
    assert K.planes_fusable(m, n)
    dz, db, planes = K.bias_act_bwd(dy, y, a, want_planes=True)
    g = _grad64(y, a)
    ref = dy.double() * g
    y64 = y.double()
    _assert_within(dz, ref, 4 * U * dy.double().abs() * (g.abs() + y64 * y64 + y64.abs()) + 1e-38, "dz")
    nblk = (m + 127) // 128
    bound_db = (128 + 8 + nblk + 32) * U * dz.double().abs().sum(0) + \
        (4 * U * dy.double().abs() * (g.abs() + y64 * y64 + y64.abs())).sum(0)
    _assert_within(db, ref.sum(0), bound_db, "dbias")
    want = _planes_ref(dz.cpu().numpy())
    got = _planes_got(planes, m, n)
    assert (got == want).all(), "%d bf16 values differ" % int((got != want).sum())
    _, db2, planes2 = K.bias_act_bwd(dy, y, a, want_dz=False, want_planes=True)
    assert torch.equal(db2, db) and torch.equal(planes2[:-256], planes[:-256])


# ---- prediction head + loss ------------------------------------------------------------------------------------
def _head_ref(z, y, task, B):
    """float64 restatement of oracle/ops.py prediction + binary_crossentropy / mse (mean over the batch) and of
    their gradient, with the kernel's fp32 eps; returns p, loss terms, dlogit, and per-element error scales"""
    z, y = z.double(), y.double()
    if task == 0:
        eps = float(np.float32(1e-7))
        hi = float(np.float32(1.0) - np.float32(1e-7))
        p = torch.sigmoid(z)
        inside = ((p >= eps) & (p <= hi)).double()

        def terms(p):
            pc = p.clamp(eps, hi)
            t1, t2 = y * torch.log(pc + eps), (1 - y) * torch.log(1 - pc + eps)
            g1, g2 = y / (pc + eps) * p * (1 - p) * inside, (1 - y) / (1 - pc + eps) * p * (1 - p) * inside
            return t1, t2, g1, g2

        t1, t2, g1, g2 = terms(p)
        # the kernel's p is within dp = 8 u p of the exact one, and that one p feeds every factor: loss and dlogit
        # are the formulas evaluated at some p' in [p - dp, p + dp] (checked at both ends; near p = 1 the eps in
        # 1 - p + eps makes dlogit steep in p), plus a few roundings of each term
        dp = 8 * U * p
        moved = [terms((p + s * dp).clamp(0, 1)) for s in (-1, 1)]
        e_l = 16 * U * (t1.abs() + t2.abs()) + torch.max(*[((a + b) - (t1 + t2)).abs() for a, b, _, _ in moved])
        e_dz = (16 * U * (g1.abs() + g2.abs()) +
                torch.max(*[((c - d) - (g1 - g2)).abs() for _, _, c, d in moved])) / B
        return p, -(t1 + t2), -(g1 - g2) / B, 8 * U * p + 1e-38, e_l, e_dz
    d = z - y
    return z, d * d, 2 * d / B, torch.zeros_like(z), 4 * U * d * d, 4 * U * (2 * d / B).abs()


@pytest.mark.parametrize("B", [1, 255, 65536, (1 << 20) + 3])
@pytest.mark.parametrize("task", ["binary", "regression"])
def test_predict_loss_float64(cuda, gen, B, task):
    """pred, dlogit, loss_sum and dbias: logits saturated on both clip branches, labels in {0, 1} and fractional,
    B large enough that the grid-stride loop iterates and the CTA partials meet in atomics"""
    L, K, _ = _mods()
    t = L.TASK_BINARY if task == "binary" else L.TASK_REGRESSION
    logit = _randn(gen, (B,), 3.0).clamp(-12, 12)
    sat = torch.tensor([40.0, -40.0, 20.0, -20.0, 100.0, -100.0, 17.5, -17.5], device=cuda)
    if B > 1:
        logit[:min(B, 8)] = sat[:min(B, 8)]
    labels = torch.where(torch.rand((B,), generator=gen, device=cuda) < 0.5,
                         (torch.rand((B,), generator=gen, device=cuda) < 0.3).float(),
                         torch.rand((B,), generator=gen, device=cuda))
    bias = torch.tensor([0.375], device=cuda)
    pred, dlogit, dbias, lsum = K.predict_loss(logit, bias, labels, t, want_grad=True)
    z = logit + bias          # the kernel's fp32 z
    p, l, dz, e_p, e_l, e_dz = _head_ref(z, labels, t, B)
    _assert_within(pred, p, e_p, "pred")
    _assert_within(dlogit, dz, e_dz + 1e-38, "dlogit")
    iters = -(-B // (min(-(-B // 256), 132 * 4) * 256))
    depth = iters + 5 + 8 + min(-(-B // 256), 132 * 4)
    _assert_within(lsum, l.sum().reshape(1), (depth * U * l.abs().sum() + e_l.sum()).reshape(1), "loss_sum")
    _assert_within(dbias, dz.sum().reshape(1), (depth * U * dz.abs().sum() + e_dz.sum()).reshape(1) + 1e-38,
                   "dbias")
    pred2, d2, b2, l2 = K.predict_loss(logit, None, None, t)
    assert d2 is None and b2 is None and l2 is None
    p2 = _head_ref(logit, labels, t, B)[0]
    _assert_within(pred2, p2, 8 * U * p2.abs() + 1e-38, "pred without bias")


# ---- optimizers ------------------------------------------------------------------------------------------------
C2_WEIGHTS = [845 * 256, 256, 256 * 128, 128, 128 * 64, 64, 64, 1]
BIG = 3000001             # more elements than one grid-stride pass covers


def _opt_state(gen, n):
    """w ~ 2^-4, g over 2^-24 .. 2^0 (tiny gradients make eps visible in Adam / Adagrad)"""
    w = _randn(gen, (n,), 2.0 ** -4)
    g = _randn(gen, (n,)) * torch.exp2(torch.randint(-24, 1, (n,), generator=gen, device=gen.device).float())
    return w, g


@pytest.mark.parametrize("l2", [0.0, 0.01])
def test_sgd_float64(cuda, gen, l2):
    """sgd_step per tensor and sgd_step_multi over 41 tensors (two launches, sizes 1 .. 3M) against float64"""
    _, K, _ = _mods()
    lr = 0.05
    sizes = C2_WEIGHTS + [BIG] + [1, 3, 5, 17, 1000, 4099] * 5 + [2]
    assert len(sizes) > 32
    ws, gs = zip(*[_opt_state(gen, s) for s in sizes])
    l2s = [l2 * (i % 3) for i in range(len(sizes))]
    lr32, l2s32 = float(np.float32(lr)), [float(np.float32(v)) for v in l2s]

    def ref(w, g, l2v):
        w, g = w.double(), g.double()
        upd = lr32 * (g + 2 * l2v * w)
        return w - upd, 4 * U * (w.abs() + lr32 * (g.abs() + 2 * l2v * w.abs())) + 1e-45

    multi = [w.clone() for w in ws]
    K.sgd_step_multi(multi, list(gs), lr, l2s)
    for i, (w, g) in enumerate(zip(ws, gs)):
        want, bound = ref(w, g, l2s32[i])
        _assert_within(multi[i], want, bound, "sgd_step_multi tensor %d (n=%d)" % (i, sizes[i]))
        if sizes[i] in C2_WEIGHTS + [BIG] and i < 9:
            one = w.clone()
            K.sgd_step(one, g, lr, l2s[i])
            _assert_within(one, want, bound, "sgd_step n=%d" % sizes[i])


def _adam_ref(w, g, m, v, lr, step, l2, b1=0.9, b2=0.999, eps=1e-7):
    """one Keras Adam step in float64 from the fp32 state, with the kernel's fp32 constants; returns values and
    error bounds of (w, m, v)"""
    f = lambda x: float(np.float32(x))
    lr, b1, b2, eps, l2 = f(lr), f(b1), f(b2), f(eps), f(l2)
    w, g, m, v = w.double(), g.double(), m.double(), v.double()
    lr_t = lr * np.sqrt(1.0 - b2 ** step) / (1.0 - b1 ** step)
    gi = g + 2 * l2 * w
    e_gi = 2 * U * (g.abs() + 2 * l2 * w.abs())
    m1 = b1 * m + (1 - b1) * gi
    e_m = 3 * U * (b1 * m.abs() + (1 - b1) * gi.abs()) + (1 - b1) * e_gi
    v1 = b2 * v + (1 - b2) * gi * gi
    e_v = 4 * U * (b2 * v + (1 - b2) * gi * gi) + (1 - b2) * 2 * gi.abs() * e_gi
    s = v1.sqrt()
    den = s + eps
    upd = lr_t * m1 / den
    e_den = torch.where(s > 0, e_v / (2 * s.clamp_min(1e-300)), e_v.sqrt()) + 2 * U * den
    e_upd = lr_t * (e_m / den + m1.abs() * e_den / (den * den)) + 6 * U * upd.abs()
    w1 = w - upd
    return (w1, m1, v1), (2 * U * w1.abs() + e_upd + 1e-45, e_m + 1e-45, e_v + 1e-45)


@pytest.mark.parametrize("l2", [0.0, 1e-4])
@pytest.mark.parametrize("dev", [False, True], ids=["adam_step", "adam_step_dev"])
def test_adam_float64_per_step(cuda, gen, l2, dev):
    """25 steps and then a jump to step 10^6 (bias correction ~ 1), each step checked against a float64 step taken
    from the same fp32 state; C2 weight sizes and a 3M-element vector"""
    _, K, _ = _mods()
    lr = 1e-3
    for n in C2_WEIGHTS[:2] + [1, BIG]:
        w, g0 = _opt_state(gen, n)
        m, v = torch.zeros(n, device=cuda), torch.zeros(n, device=cuda)
        ctr = torch.zeros(1, dtype=torch.int64, device=cuda)
        for step in list(range(1, 26)) + [10 ** 6]:
            g = g0 * (1.0 + 0.1 * (step % 7)) if step < 100 else -g0
            (w1, m1, v1), (ew, em, ev) = _adam_ref(w, g, m, v, lr, step, l2)
            if dev:
                K.counter_add(ctr, step - int(ctr.item()))
                K.adam_step_dev(w, g, m, v, lr, ctr, l2=l2)
            else:
                K.adam_step(w, g, m, v, lr, step, l2=l2)
            _assert_within(m, m1, em, "m step %d n=%d" % (step, n))
            _assert_within(v, v1, ev, "v step %d n=%d" % (step, n))
            _assert_within(w, w1, ew, "w step %d n=%d" % (step, n))


@pytest.mark.parametrize("l2", [0.0, 1e-4])
def test_adagrad_float64_per_step(cuda, gen, l2):
    _, K, _ = _mods()
    lr, eps = 0.01, 1e-7
    f = lambda x: float(np.float32(x))
    for n in C2_WEIGHTS[:2] + [BIG]:
        w, g0 = _opt_state(gen, n)
        acc = torch.full((n,), 0.1, device=cuda)
        for step in range(1, 6):
            g = g0 * step
            w64, g64, a64 = w.double(), g.double(), acc.double()
            gi = g64 + 2 * f(l2) * w64
            e_gi = 2 * U * (g64.abs() + 2 * f(l2) * w64.abs())
            a1 = a64 + gi * gi
            e_a = 2 * U * a1 + 2 * gi.abs() * e_gi
            den = a1.sqrt() + f(eps)
            upd = f(lr) * gi / den
            e_upd = f(lr) * (e_gi / den + gi.abs() * (e_a / (2 * a1.sqrt()) + 2 * U * den) / (den * den)) + \
                6 * U * upd.abs()
            K.adagrad_step(w, g, acc, lr, eps, l2)
            _assert_within(acc, a1, e_a, "acc step %d" % step)
            _assert_within(w, w64 - upd, 2 * U * (w64 - upd).abs() + e_upd + 1e-45, "w step %d" % step)


# ---- unfused FM and the plumbing kernels -----------------------------------------------------------------------
@pytest.mark.parametrize("E", [32, 40])
def test_fm_window_exact(cuda, gen, E):
    """fm_fwd / fm_bwd at B = 65536, F = 26 on a column window of the DNN input buffer (after 13 dense columns),
    the gradient accumulated into the same window of a gradient buffer; exact-valued, so equal to float64"""
    _, K, _ = _mods()
    B, F = 65536, 26
    ld = (13 + F * E + 3 + 3) // 4 * 4
    xb = torch.full((B, ld), float("nan"), device=cuda)
    xb[:, 13:13 + F * E] = _ints(gen, (B, F * E), -8, 8, 2.0 ** -4)
    x = xb[:, 13:13 + F * E]
    x64 = x.double().reshape(B, F, E)
    s = x64.sum(1)
    want = 0.5 * (s * s - (x64 * x64).sum(1)).sum(1)
    _exact_ok(0.5 * ((x64.abs().sum(1)) ** 2 + (x64 * x64).sum(1)).sum(1), 2.0 ** -8)
    _assert_equal(K.fm_fwd(x, F, E), want, "fm_fwd")
    g = _ints(gen, (B,), -8, 8, 2.0 ** -4)
    db = torch.full((B, ld), 9.0, device=cuda)
    d0 = _ints(gen, (B, F * E), -64, 64, 2.0 ** -8)
    db[:, 13:13 + F * E] = d0
    K.fm_bwd(x, F, E, g, dx=db[:, 13:13 + F * E], accumulate=True)
    dref = d0.double() + (g.double()[:, None, None] * (s[:, None, :] - x64)).reshape(B, F * E)
    _assert_equal(db[:, 13:13 + F * E], dref, "fm_bwd accumulate")
    assert bool((db[:, :13] == 9.0).all()) and bool((db[:, 13 + F * E:] == 9.0).all())
    fresh = K.fm_bwd(x, F, E, g)
    _assert_equal(fresh, dref - d0.double(), "fm_bwd")


def test_rowsum_copy2d_add_n_act_exact(cuda, gen):
    """C2 sizes: rowsum of the [B, 845] window, copy2d in the float4 and scalar paths with accumulate, add_n with
    1 .. 8 inputs, act_fwd (relu exact; sigmoid / tanh within a few ulps of float64)"""
    L, K, _ = _mods()
    B = 65536
    xb, x = _padded(gen, B, 845, 848, float("nan"), -8, 8, 2.0 ** -4)
    _assert_equal(K.rowsum(x, B, 845), x.double().sum(1), "rowsum")
    # copy2d: [B, 256] into columns 4..260 of a [B, 848] buffer (float4), then [B, 845] window -> offset 1 (scalar)
    src = _ints(gen, (B, 256), -8, 8, 2.0 ** -4)
    dst = _ints(gen, (B, 848), -8, 8, 2.0 ** -4)
    d0 = dst.clone()
    K.copy2d(src, 256, dst, 848, B, 256, accumulate=True, dst_off=4)
    want = d0.double()
    want[:, 4:260] += src.double()
    _assert_equal(dst, want, "copy2d float4 accumulate")
    K.copy2d(src, 256, dst, 848, B, 256, dst_off=300)
    want[:, 300:556] = src.double()
    _assert_equal(dst, want, "copy2d float4")
    dst2 = _ints(gen, (B, 850), -8, 8, 2.0 ** -4)
    e0 = dst2.clone()
    K.copy2d(xb, 848, dst2, 850, B, 845, accumulate=True, dst_off=1)
    want2 = e0.double()
    want2[:, 1:846] += x.double()
    _assert_equal(dst2, want2, "copy2d scalar accumulate")
    # add_n
    ins = [_ints(gen, (B, 256), -8, 8, 2.0 ** -4) for _ in range(8)]
    scales = [1.0, -2.0, 0.5, 0.25, -1.0, 4.0, -0.125, 2.0]
    for nin in range(1, 9):
        got = K.add_n(ins[:nin], scales=scales[:nin])
        _assert_equal(got, sum(s * t.double() for s, t in zip(scales[:nin], ins[:nin])), "add_n %d" % nin)
    # act_fwd
    z = _randn(gen, (B, 256), 4.0)
    _assert_equal(K.act_fwd(z, L.ACT_RELU), torch.relu(z.double()), "relu")
    for a, f in ((L.ACT_SIGMOID, torch.sigmoid), (L.ACT_TANH, torch.tanh)):
        ref = f(z.double())
        _assert_within(K.act_fwd(z, a), ref, 8 * U * ref.abs() + 1e-38, "act %d" % a)


# ---- one composed tower through ops.dense ----------------------------------------------------------------------
def test_dense_tower_composed(cuda, gen, gemm_precision):
    """ops.dense with relu, 845 -> 256 -> 128 -> 64 -> 1 (linear) at B = 65536 on the [B, 845] window of a
    [B, 848] buffer (pad columns NaN): the forward and the x, W, b gradients against float64.  The backward
    reference takes the relu masks from the kernels' own activations (the forward is checked separately), and the
    bounds follow the error of each GEMM through |W| and the 1-Lipschitz relu."""
    from deepctr_b200 import engine as E
    L, K, ops = _mods()
    B, dims = 65536, [845, 256, 128, 64, 1]
    xb = torch.full((B, 848), float("nan"), device=cuda)
    xb[:, :845] = _randn(gen, (B, 845))
    base = E.Var(xb, requires_grad=True)
    x = ops._window(base, 0, 845, (B, 845))
    Ws = [E.Var(_randn(gen, (dims[i], dims[i + 1]), dims[i] ** -0.5), requires_grad=True) for i in range(4)]
    bs = [E.Var(_randn(gen, (dims[i + 1],), 0.1), requires_grad=True) for i in range(4)]
    tape = E.Tape()
    hs = [x]
    with E.recording(tape):
        for i in range(4):
            hs.append(ops.dense(hs[-1], Ws[i], bs[i], activation="relu" if i < 3 else None))
    gy = _randn(gen, (B, 1))
    hs[-1].requires_grad = True
    E.add_grad(hs[-1], gy)
    tape.backward()
    torch.cuda.synchronize()

    def eps(k, n, splits=1):            # relative error of one GEMM in the precision ops.dense picks for it
        e = (k + splits + 8) * U
        if gemm_precision == "bf16x3" and min(n, k) >= 16 and k >= 16:
            e += 2.0 ** -15
        return e

    # forward: ref, |.|-chain, error chain
    h64, habs, err = xb[:, :845].double(), xb[:, :845].double().abs(), None
    for i in range(4):
        W, b = Ws[i].data.double(), bs[i].data.double()
        pre = h64 @ W + b
        a = habs @ W.abs() + b.abs()
        e_i = eps(dims[i], dims[i + 1]) * a + (err @ W.abs() if err is not None else 0.0)
        h64, habs, err = (torch.relu(pre) if i < 3 else pre), a, e_i
        got = hs[i + 1].data.reshape(B, dims[i + 1])
        _assert_within(got, h64, err + 1e-30, "forward layer %d (%s)" % (i + 1, gemm_precision))
    # backward from the kernels' activations
    acts = [xb[:, :845]] + [hs[i].data.reshape(B, dims[i]) for i in range(1, 5)]
    g64, gabs, gerr = gy.double(), gy.double().abs(), torch.zeros_like(gy, dtype=torch.float64)
    for i in reversed(range(4)):
        W = Ws[i].data.double()
        mask = (acts[i + 1] > 0).double() if i < 3 else torch.ones_like(g64)
        dz, dzabs, dzerr = g64 * mask, gabs * mask, gerr * mask
        hin = acts[i].double()
        k_red = B
        sk = ops._split_k(dims[i], dims[i + 1], B)
        e_w = eps(k_red // sk + 1, dims[i + 1], sk) if dims[i + 1] >= 16 or gemm_precision == "fp32" else \
            (k_red // sk + sk + 24) * U
        if gemm_precision == "bf16x3" and min(dims[i], dims[i + 1]) >= 16:
            e_w = (k_red // sk + sk + 8) * U + 2.0 ** -15
        bw = e_w * (hin.abs().t() @ dzabs) + hin.abs().t() @ dzerr
        _assert_within(Ws[i].grad, hin.t() @ dz, bw + 1e-30, "dW layer %d (%s)" % (i + 1, gemm_precision))
        nblk = (B + 127) // 128
        bb = (128 + 8 + nblk + 32) * U * dzabs.sum(0) + dzerr.sum(0)
        _assert_within(bs[i].grad.reshape(-1), dz.sum(0), bb + 1e-30, "db layer %d (%s)" % (i + 1, gemm_precision))
        g64 = dz @ W.t()
        e_d = eps(dims[i + 1], dims[i]) if min(dims[i], dims[i + 1]) >= 16 else (dims[i + 1] + 8) * U
        gabs = dzabs @ W.abs().t()
        gerr = e_d * gabs + dzerr @ W.abs().t()
    got_dx = base.grad[:, :845]
    _assert_within(got_dx, g64, gerr + 1e-30, "dx (%s)" % gemm_precision)
