"""GPU parity: GEMM / elementwise / FM / head / optimizer kernels through the C-ABI vs torch-CPU fp32."""
import numpy as np
import pytest
import torch

from oracle import ops as O

pytestmark = pytest.mark.gpu


def _kern():
    from deepctr_b200 import kernels as K, _lib as L
    return K, L


def _r(rng, *shape):
    return torch.tensor(rng.normal(size=shape).astype(np.float32))


@pytest.mark.parametrize("m,n,k", [(1, 1, 1), (257, 256, 845), (130, 64, 128), (1000, 1, 64),
                                   (64, 300, 7)])
@pytest.mark.parametrize("ta,tb", [(False, False), (False, True), (True, False), (True, True)])
def test_gemm_fp32_layouts(cuda, m, n, k, ta, tb):
    K, L = _kern()
    rng = np.random.RandomState(m * 7 + n)
    a = _r(rng, *((k, m) if ta else (m, k)))
    b = _r(rng, *((n, k) if tb else (k, n)))
    bias = _r(rng, n)
    want = torch.relu((a.t() if ta else a).double() @ (b.t() if tb else b).double() + bias.double()).float()
    got = K.gemm(a.to(cuda), b.to(cuda), bias=bias.to(cuda), trans_a=ta, trans_b=tb, act=L.ACT_RELU, m=m, n=n, k=k)
    torch.testing.assert_close(got.cpu(), want, rtol=1e-4, atol=1e-4)


@pytest.mark.parametrize("m,n,k", [(5000, 3, 70), (4096, 8, 64), (3000, 5, 16), (2049, 64, 1), (1000, 17, 8),
                                   (65536, 1, 64), (777, 2, 1000), (33, 1, 19)])
@pytest.mark.parametrize("tb", [False, True])
def test_gemm_fp32_skinny_shapes(cuda, m, n, k, tb):
    """GEMV (N <= 8) and outer-product (K <= 8) kernels behind the same b2ctr_gemm entry point: the last
    [*, 1] projection of every tower and its dgrad; strided A / C, alpha, accumulate, bias + activation."""
    K, L = _kern()
    rng = np.random.RandomState(m + n + k)
    a_wide = _r(rng, m, k + 4).to(cuda)
    a = a_wide[:, :k]                                   # lda = k + 4
    b = _r(rng, *((n, k) if tb else (k, n))).to(cuda)
    bias = _r(rng, n).to(cuda)
    A, Bm = a.cpu().double(), (b.t() if tb else b).cpu().double()
    got = K.gemm(a, b, bias=bias, trans_b=tb, act=L.ACT_TANH, m=m, n=n, k=k)
    want = torch.tanh(A @ Bm + bias.cpu().double()).float()
    torch.testing.assert_close(got.cpu(), want, rtol=1e-4, atol=1e-4)
    c_wide = _r(rng, m, n + 3).to(cuda)
    c0 = c_wide.clone()
    K.gemm(a, b, c=c_wide[:, :n], trans_b=tb, accumulate=True, alpha=0.25, m=m, n=n, k=k)
    want2 = c0.cpu().double()
    want2[:, :n] += 0.25 * (A @ Bm)
    torch.testing.assert_close(c_wide.cpu(), want2.float(), rtol=1e-4, atol=1e-4)   # columns >= n untouched


@pytest.mark.parametrize("m,n,k,sk", [(64, 1, 65536, 74), (13, 1, 65536, 74), (845, 3, 9000, 4), (64, 1, 200, 1),
                                      (100, 8, 4097, 5), (1, 1, 70000, 64)])
@pytest.mark.parametrize("tb", [False, True])
def test_gemm_fp32_skinny_wgrad(cuda, m, n, k, sk, tb):
    """A stored [K, M] with N <= 8 (wgrad of the [*, 1] projections): streaming reduction over the batch,
    K slices through the split-K workspace."""
    K, L = _kern()
    rng = np.random.RandomState(m + n + k)
    a_wide = _r(rng, k, m + 4).to(cuda)
    a = a_wide[:, :m]
    b = _r(rng, *((n, k) if tb else (k, n))).to(cuda)
    c0 = _r(rng, m, n)
    want = c0.double() + 0.5 * (a.cpu().double().t() @ (b.t() if tb else b).cpu().double())
    c = c0.to(cuda)
    K.gemm(a, b, c=c, trans_a=True, trans_b=tb, accumulate=True, alpha=0.5, split_k=sk, m=m, n=n, k=k)
    torch.testing.assert_close(c.cpu(), want.float(), rtol=1e-4, atol=2e-3 * max(1.0, (k / 256.0) ** 0.5))


def test_gemm_splitk_accumulate_and_ld(cuda):
    K, L = _kern()
    rng = np.random.RandomState(3)
    m, n, k = 845, 256, 4099          # wgrad shape: reduction over the batch
    x = _r(rng, k, 848)[:, :m]        # stored [K, M] with ld 848 (K-padded activations)
    dy = _r(rng, k, n)
    c0 = _r(rng, m, n)
    want = (c0.double() + 0.5 * (x.t().double() @ dy.double())).float()
    xd = _r(rng, k, 848).to(cuda)
    xd[:, :m] = x.to(cuda)
    c = c0.to(cuda)
    K.gemm(xd, dy.to(cuda), c=c, trans_a=True, accumulate=True, split_k=16, alpha=0.5, m=m, n=n, k=k)
    torch.testing.assert_close(c.cpu(), want, rtol=1e-4, atol=2e-4)
    # determinism of the split-K reduction
    c2 = c0.to(cuda)
    K.gemm(xd, dy.to(cuda), c=c2, trans_a=True, accumulate=True, split_k=16, alpha=0.5, m=m, n=n, k=k)
    assert torch.equal(c, c2)


def test_gemm_rejects_bad_arguments(cuda):
    K, L = _kern()
    a = torch.zeros((4, 4), device=cuda)
    with pytest.raises(ValueError):
        K.gemm(a, a, act=L.ACT_RELU, accumulate=True)
    with pytest.raises(ValueError):
        K.gemm(a, a, precision=99)


@pytest.mark.parametrize("act", ["relu", "sigmoid", "tanh", None])
def test_bias_act_bwd(cuda, act):
    K, L = _kern()
    rng = np.random.RandomState(4)
    m, n = 1031, 200
    z = _r(rng, m, n).requires_grad_(True)
    y = O._ACT[act](z)
    dy = _r(rng, m, n)
    (y * dy).sum().backward()
    dz, db = K.bias_act_bwd(dy.to(cuda), y.detach().to(cuda), L.ACT_BY_NAME[act])
    torch.testing.assert_close(dz.cpu(), z.grad, rtol=1e-5, atol=1e-6)
    torch.testing.assert_close(db.cpu(), z.grad.sum(0), rtol=1e-4, atol=1e-4)


def test_act_fwd_add_axpy_copy_rowsum_fill(cuda):
    K, L = _kern()
    rng = np.random.RandomState(5)
    x = _r(rng, 1000, 37)
    xd = x.to(cuda)
    for name in ["relu", "sigmoid", "tanh"]:
        torch.testing.assert_close(K.act_fwd(xd, L.ACT_BY_NAME[name]).cpu(), O._ACT[name](x),
                                   rtol=1e-6, atol=1e-6)
    y = _r(rng, 1000, 37)
    got = K.add_n([xd, y.to(cuda), xd], scales=[1.0, -2.0, 0.5]).cpu()
    torch.testing.assert_close(got, 1.5 * x - 2 * y, rtol=1e-6, atol=1e-6)
    yd = y.to(cuda)
    K.axpy(xd, yd, 0.25)
    torch.testing.assert_close(yd.cpu(), y + 0.25 * x, rtol=1e-6, atol=1e-6)
    # concat two blocks into a wider buffer, then slice-accumulate back
    dst = torch.zeros((1000, 80), device=cuda)
    K.copy2d(xd, 37, dst, 80, 1000, 37, dst_off=4)
    assert torch.equal(dst[:, 4:41].cpu(), x)
    K.copy2d(dst, 80, xd, 37, 1000, 37, accumulate=True, src_off=4)
    assert torch.equal(xd.cpu(), 2 * x)
    v4 = _r(rng, 64, 32).to(cuda)
    dst4 = torch.zeros((64, 64), device=cuda)
    K.copy2d(v4, 32, dst4, 64, 64, 32, dst_off=32)
    assert torch.equal(dst4[:, 32:], v4)
    torch.testing.assert_close(K.rowsum(v4, 64, 32).cpu(), v4.cpu().sum(1), rtol=1e-5, atol=1e-5)
    f = torch.empty(1001, device=cuda)
    K.fill(f, 3.5)
    assert torch.all(f == 3.5)


@pytest.mark.parametrize("F,E", [(26, 32), (4, 3), (7, 40)])
def test_fm_fwd_bwd(cuda, F, E):
    K, L = _kern()
    rng = np.random.RandomState(6)
    B = 333
    x = _r(rng, B, F, E).requires_grad_(True)
    out = O.fm(x)
    g = _r(rng, B)
    (out[:, 0] * g).sum().backward()
    xd = x.detach().reshape(B, F * E).to(cuda)
    torch.testing.assert_close(K.fm_fwd(xd, F, E).cpu(), out[:, 0].detach(), rtol=1e-4, atol=1e-4)
    dx = K.fm_bwd(xd, F, E, g.to(cuda))
    torch.testing.assert_close(dx.cpu().reshape(B, F, E), x.grad, rtol=1e-4, atol=1e-4)
    # closed form of SURVEY.md section 8c: FM == sum_{i<j} <v_i, v_j>
    xx = x.detach().double()
    pair = sum((xx[:, i] * xx[:, j]).sum(-1) for i in range(F) for j in range(i + 1, F))
    torch.testing.assert_close(K.fm_fwd(xd, F, E).cpu().double(), pair, rtol=1e-4, atol=1e-4)


@pytest.mark.parametrize("task", ["binary", "regression"])
def test_predict_loss(cuda, task):
    K, L = _kern()
    rng = np.random.RandomState(7)
    B = 4097
    logit = (_r(rng, B) * 3).requires_grad_(True)
    logit.data[0], logit.data[1] = 40.0, -40.0      # saturated: exercises the clip branch
    bias = torch.tensor([0.3], requires_grad=True)
    y = torch.tensor((rng.rand(B) < 0.25).astype(np.float32))
    p = O.prediction(logit[:, None], bias, task)
    loss = O.binary_crossentropy(y, p) if task == "binary" else O.mse(y, p)
    loss.backward()
    t = L.TASK_BINARY if task == "binary" else L.TASK_REGRESSION
    pred, dlogit, dbias, lsum = K.predict_loss(logit.detach().to(cuda), bias.detach().to(cuda), y.to(cuda),
                                               t, want_grad=True)
    torch.testing.assert_close(pred.cpu(), p.detach()[:, 0], rtol=1e-5, atol=1e-6)
    torch.testing.assert_close(lsum.cpu() / B, loss.detach().reshape(1), rtol=1e-4, atol=1e-6)
    torch.testing.assert_close(dlogit.cpu(), logit.grad, rtol=1e-4, atol=1e-9)
    torch.testing.assert_close(dbias.cpu(), bias.grad, rtol=1e-3, atol=1e-7)
    pred2, _, _, _ = K.predict_loss(logit.detach().to(cuda), None, None, t)
    torch.testing.assert_close(pred2.cpu(), O.prediction(logit.detach()[:, None], None, task)[:, 0],
                               rtol=1e-5, atol=1e-6)


def test_optimizers(cuda):
    K, L = _kern()
    rng = np.random.RandomState(8)
    n = 5003
    w0, g = _r(rng, n), _r(rng, n)
    # SGD (+ l2: d/dw l2*w^2 = 2*l2*w, Keras regularizers.l2)
    w = w0.to(cuda)
    K.sgd_step(w, g.to(cuda), 0.1, 0.01)
    torch.testing.assert_close(w.cpu(), w0 - 0.1 * (g + 0.02 * w0), rtol=1e-6, atol=1e-6)
    # the multi-tensor form (one launch for all the dense weights of a tower): bit-identical to the per-tensor kernel
    sizes = [1, 7, 256, 5003, 40000] * 8                       # 40 tensors: two launches of <= 32
    ws0 = [_r(rng, k) for k in sizes]
    gs = [_r(rng, k) for k in sizes]
    l2s = [0.0 if i % 2 else 0.01 for i in range(len(sizes))]
    one = [t.to(cuda) for t in ws0]
    many = [t.to(cuda) for t in ws0]
    gd = [t.to(cuda) for t in gs]
    for t, gg, l2 in zip(one, gd, l2s):
        K.sgd_step(t, gg, 0.1, l2)
    K.sgd_step_multi(many, gd, 0.1, l2s)
    for a, b in zip(one, many):
        assert torch.equal(a, b)
    # Adam: 3 steps vs torch.optim.Adam(eps=1e-7) - Keras places eps outside the bias correction
    wt = w0.clone().double()
    m = torch.zeros(n).double()
    v = torch.zeros(n).double()
    w = w0.to(cuda)
    md, vd = torch.zeros(n, device=cuda), torch.zeros(n, device=cuda)
    for step in range(1, 4):
        gs = (g * step).double()
        m = 0.9 * m + 0.1 * gs
        v = 0.999 * v + 0.001 * gs * gs
        lr_t = 1e-3 * np.sqrt(1 - 0.999 ** step) / (1 - 0.9 ** step)
        wt = wt - lr_t * m / (v.sqrt() + 1e-7)
        K.adam_step(w, (g * step).to(cuda), md, vd, 1e-3, step)
    torch.testing.assert_close(w.cpu().double(), wt, rtol=1e-5, atol=1e-6)
    # Adagrad
    w = w0.to(cuda)
    acc = torch.full((n,), 0.1, device=cuda)
    K.adagrad_step(w, g.to(cuda), acc, 0.01)
    a = 0.1 + g * g
    torch.testing.assert_close(w.cpu(), w0 - 0.01 * g / (a.sqrt() + 1e-7), rtol=1e-5, atol=1e-6)


@pytest.mark.parametrize("m,n,k", [(128, 128, 64), (1, 1, 1), (257, 256, 845), (130, 64, 128), (1000, 1, 64),
                                   (64, 300, 7), (4096, 256, 848), (300, 40, 200)])
@pytest.mark.parametrize("ta,tb", [(False, False), (False, True), (True, False), (True, True)])
@pytest.mark.parametrize("variant", [3, 4])
def test_gemm_bf16x3_tensor_core(cuda, m, n, k, ta, tb, variant):
    """wgmma split-bf16 GEMM: a = hi_a + lo_a and b = hi_b + lo_b in bf16, and the product drops only lo_a lo_b, at most
    2^-16 |a||b| per term (DESIGN.md section 5); 2^-15 sum |a||b| also covers the fp32 accumulation at these k.
    Variants: 3 = non-persistent reference kernel, 4 = persistent warp-specialised kernel."""
    K, L = _kern()
    rng = np.random.RandomState(m + 3 * n + k)
    a = _r(rng, *((k, m) if ta else (m, k)))
    b = _r(rng, *((n, k) if tb else (k, n)))
    bias = _r(rng, n)
    A = (a.t() if ta else a).double()
    Bm = (b.t() if tb else b).double()
    want = torch.relu(A @ Bm + bias.double())
    got = K.gemm(a.to(cuda), b.to(cuda), bias=bias.to(cuda), trans_a=ta, trans_b=tb, act=L.ACT_RELU,
                 precision=L.GEMM_BF16X3, m=m, n=n, k=k, variant=variant).cpu().double()
    bound = (A.abs() @ Bm.abs()) * 2.0 ** -15 + 1e-6
    assert ((got - want).abs() <= bound).all(), float(((got - want).abs() / bound).max())


@pytest.mark.parametrize("m,n,k", [(128, 128, 64), (257, 256, 845), (4096, 256, 848), (300, 40, 200), (1000, 1, 64),
                                   (845, 256, 4100), (4096, 845, 256), (515, 384, 130)])
@pytest.mark.parametrize("ta,tb", [(False, False), (False, True), (True, False), (True, True)])
@pytest.mark.parametrize("given", ["a", "b", "ab"])
@pytest.mark.parametrize("variant", [3, 4])
def test_gemm_bf16x3_with_caller_planes(cuda, m, n, k, ta, tb, given, variant):
    """b2ctr_split_planes output handed to b2ctr_gemm (a_planes / b_planes) must give the same result as
    the GEMM splitting its operands itself: the planes are a pure function of the stored matrix."""
    K, L = _kern()
    rng = np.random.RandomState(m + 3 * n + k)
    a = _r(rng, *((k, m) if ta else (m, k))).to(cuda)
    b = _r(rng, *((n, k) if tb else (k, n))).to(cuda)
    ap = K.split_planes(a) if "a" in given else None
    bp = K.split_planes(b) if "b" in given else None
    sk = 4 if k > 2048 else 1
    want = K.gemm(a, b, trans_a=ta, trans_b=tb, precision=L.GEMM_BF16X3, m=m, n=n, k=k, split_k=sk, variant=variant)
    got = K.gemm(a, b, trans_a=ta, trans_b=tb, precision=L.GEMM_BF16X3, m=m, n=n, k=k, split_k=sk, variant=variant,
                 a_planes=ap, b_planes=bp)
    assert torch.equal(want, got)
    # strided source (leading window of a wider buffer), as ops.dense passes the embedding concat buffer
    wide = torch.zeros((a.shape[0], a.shape[1] + 5), device=cuda)
    wide[:, :a.shape[1]] = a
    got2 = K.gemm(wide[:, :a.shape[1]], b, trans_a=ta, trans_b=tb, precision=L.GEMM_BF16X3, m=m, n=n, k=k,
                  split_k=sk, variant=variant, a_planes=K.split_planes(wide[:, :a.shape[1]]), b_planes=bp)
    assert torch.equal(want, got2)


@pytest.mark.parametrize("m,n,k,ta,tb,sk", [(40000, 256, 845, False, False, 1), (40000, 845, 256, False, True, 1),
                                             (845, 256, 40000, True, False, 18), (30000, 128, 256, False, False, 1),
                                             (30000, 64, 128, False, True, 1), (20000, 40, 100, False, False, 1),
                                             (256, 256, 30000, True, False, 37)])
def test_gemm_bf16x3_persistent_pair_many_tiles(cuda, m, n, k, ta, tb, sk):
    """Variant 4 at shapes where every CTA walks many tiles (the producers run ahead across tile boundaries, several trips
    round the stage ring): same products in the same K order as the one-tile-per-CTA kernel -> identical."""
    K, L = _kern()
    rng = np.random.RandomState(m + n + k)
    a = _r(rng, *((k, m) if ta else (m, k))).to(cuda)
    b = _r(rng, *((n, k) if tb else (k, n))).to(cuda)
    bias = _r(rng, n).to(cuda)
    kw = dict(trans_a=ta, trans_b=tb, precision=L.GEMM_BF16X3, m=m, n=n, k=k, split_k=sk)
    if sk == 1:
        kw.update(bias=bias, act=L.ACT_RELU)
    want = K.gemm(a, b, variant=3, **kw)
    for _ in range(3):
        got = K.gemm(a, b, variant=4, **kw)
        assert torch.equal(want, got), float((want - got).abs().max())
    ref = K.gemm(a, b, **{**kw, "precision": L.GEMM_FP32})
    torch.testing.assert_close(got, ref, rtol=2e-4, atol=2e-3 * max(1.0, (k / 256.0) ** 0.5))


@pytest.mark.parametrize("variant", [3, 4])
def test_gemm_bf16x3_splitk_accumulate(cuda, variant):
    K, L = _kern()
    rng = np.random.RandomState(77)
    m, n, k = 845, 256, 8200
    xd = _r(rng, k, 848).to(cuda)
    dy = _r(rng, k, n).to(cuda)
    c0 = _r(rng, m, n)
    want = c0.double() + 0.5 * (xd.cpu()[:, :m].t().double() @ dy.cpu().double())
    c = c0.to(cuda)
    K.gemm(xd, dy, c=c, trans_a=True, accumulate=True, split_k=8, alpha=0.5, precision=L.GEMM_BF16X3,
           m=m, n=n, k=k, variant=variant)
    bound = (xd.cpu()[:, :m].t().double().abs() @ dy.cpu().double().abs()) * 2.0 ** -15 + 1e-5
    assert ((c.cpu().double() - want).abs() <= bound).all()
    # against the exact-fp32 path on the same inputs
    c2 = c0.to(cuda)
    K.gemm(xd, dy, c=c2, trans_a=True, accumulate=True, split_k=8, alpha=0.5, m=m, n=n, k=k)
    torch.testing.assert_close(c.cpu(), c2.cpu(), rtol=1e-4, atol=2e-3)


@pytest.mark.parametrize("variant", [1, 2, 5])
def test_gemm_bf16x3_rejects_unknown_variant(cuda, variant):
    """only 0 (default), 3 and 4 select a kernel; anything else is an argument error and launches nothing"""
    K, L = _kern()
    a, b = torch.ones((256, 64), device=cuda), torch.ones((64, 128), device=cuda)
    n0 = L.launch_count()
    with pytest.raises(ValueError, match="variant"):
        K.gemm(a, b, precision=L.GEMM_BF16X3, variant=variant)
    assert L.launch_count() == n0


@pytest.mark.parametrize("given", ["a", "b"])
def test_gemm_bf16x3_rejects_misaligned_planes(cuda, given):
    """caller planes must be 16-byte aligned (TMA and cp.async read them in 16-byte units): a view 8 bytes into an
    allocation is an argument error and launches nothing"""
    K, L = _kern()
    a, b = torch.ones((256, 64), device=cuda), torch.ones((64, 128), device=cuda)
    planes = K.split_planes(a if given == "a" else b)
    buf = torch.zeros(planes.numel() + 8, dtype=torch.uint8, device=cuda)
    buf[8:].copy_(planes)
    n0 = L.launch_count()
    with pytest.raises(ValueError, match="aligned"):
        K.gemm(a, b, precision=L.GEMM_BF16X3, **{given + "_planes": buf[8:]})
    assert L.launch_count() == n0


@pytest.mark.parametrize("m,n", [(512, 256), (256, 128), (1024, 64)])
def test_bias_act_bwd_emits_operand_planes(cuda, m, n):
    """b2ctr_bias_act_bwd_planes: dz, dbias unchanged, planes identical to b2ctr_split_planes(dz)."""
    K, L = _kern()
    rng = np.random.RandomState(m + n)
    dy, y = _r(rng, m, n).to(cuda), torch.relu(_r(rng, m, n)).to(cuda)
    dz0, db0 = K.bias_act_bwd(dy, y, L.ACT_RELU)
    assert K.planes_fusable(m, n) and not K.planes_fusable(m + 1, n) and not K.planes_fusable(m, 96)
    dz, db, planes = K.bias_act_bwd(dy, y, L.ACT_RELU, want_planes=True)
    assert torch.equal(dz, dz0) and torch.equal(db, db0)
    want = K.split_planes(dz0)
    assert torch.equal(planes[:-256], want[:-256])
    with pytest.raises(ValueError):
        K.bias_act_bwd(dy[:m - 1], y[:m - 1], L.ACT_RELU, want_planes=True)


def test_adam_step_with_device_step_counter(cuda):
    """b2ctr_adam_step_dev + b2ctr_counter_add == b2ctr_adam_step with the step passed by value."""
    K, L = _kern()
    rng = np.random.RandomState(8)
    n = 5000
    w0, g = _r(rng, n), _r(rng, n)
    wa, wb = w0.to(cuda), w0.to(cuda)
    ma, va = torch.zeros(n, device=cuda), torch.zeros(n, device=cuda)
    mb, vb = torch.zeros(n, device=cuda), torch.zeros(n, device=cuda)
    ctr = torch.zeros(1, dtype=torch.int64, device=cuda)
    for step in range(1, 6):
        gs = (g * step).to(cuda)
        K.adam_step(wa, gs, ma, va, 1e-3, step, l2=1e-4)
        K.counter_add(ctr, 1)
        K.adam_step_dev(wb, gs, mb, vb, 1e-3, ctr, l2=1e-4)
        assert int(ctr.item()) == step
        torch.testing.assert_close(wb, wa, rtol=1e-6, atol=1e-8)
    assert torch.equal(ma, mb) and torch.equal(va, vb)
