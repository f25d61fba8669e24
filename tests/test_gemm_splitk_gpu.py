"""GPU: split-K launches of the persistent split-bf16 GEMM (the DNN tower's weight gradients).

Their slices leave through the TMA epilogue into a [splits, m, n] workspace, launches with at most one unit per CTA
run both consumer warpgroups on it, and the float4 reduction adds the slices in the scalar kernel's order.  Variant 3
(non-persistent kernel, register epilogue, scalar reduction) is the reference: variant 0 must equal it bit for bit.
Also: ops.dense's backward gives the same gradients without writing the fp32 dz it never reads."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def _mods():
    from deepctr_b200 import _lib as L, kernels as K, ops
    return L, K, ops


def _wgrad(cuda, kin, nout, B, sk, accumulate=False, alpha=1.0, bias=False, relu=False):
    """dW[kin, nout] = act(alpha X^T dZ [+ dW] [+ bias]) from MN-major planes, as ops.dense passes them; X is the
    leading window of a [B, ld] buffer with ld a multiple of 4.  Returns (variant 0, variant 3)."""
    L, K, _ = _mods()
    rng = np.random.RandomState(kin + 3 * nout + sk)
    ld = (kin + 3) // 4 * 4
    xw = torch.tensor(rng.normal(size=(B, ld)).astype(np.float32)).to(cuda)
    x = xw[:, :kin]
    dz = torch.tensor(rng.normal(size=(B, nout)).astype(np.float32)).to(cuda)
    bv = torch.tensor(rng.normal(size=nout).astype(np.float32)).to(cuda) if bias else None
    c0 = torch.tensor(rng.normal(size=(kin, nout)).astype(np.float32)).to(cuda)
    xp, dzp = K.split_planes(x), K.split_planes(dz)
    outs = []
    for variant in (0, 3):
        c = c0.clone() if accumulate else torch.full((kin, nout), 7.0, device=cuda)
        K.gemm(x, dz, c=c, bias=bv, trans_a=True, act=L.ACT_RELU if relu else L.ACT_NONE, accumulate=accumulate,
               alpha=alpha, precision=L.GEMM_BF16X3, split_k=sk, m=kin, n=nout, k=B, a_planes=xp, b_planes=dzp,
               variant=variant)
        outs.append(c)
    torch.cuda.synchronize()
    return outs


@pytest.mark.parametrize("kin,nout", [(845, 256), (256, 128), (128, 64)])
def test_bench_wgrads_match_variant3(cuda, kin, nout):
    """the C2 tower's three wgrads at the batch and split counts the model uses"""
    _, _, ops = _mods()
    B = 65536
    got, want = _wgrad(cuda, kin, nout, B, ops._split_k(kin, nout, B))
    assert torch.equal(got, want), float((got - want).abs().max())


@pytest.mark.parametrize("kin,nout,B,sk,kw", [
    (845, 256, 16384, 16, dict(accumulate=True, alpha=0.5)),      # accumulate into C, 252 units: ping-pong
    (256, 128, 8192, 8, dict(alpha=-2.0)),                        # cooperative, alpha != 1
    (300, 128, 8192, 8, dict(bias=True, relu=True)),              # bias + activation in the reduction, m % 128 != 0
    (128, 64, 16384, 16, dict(bias=True, accumulate=True)),       # BN = 64, cooperative
    (200, 90, 8192, 8, dict(bias=True, relu=True)),               # n % 4 != 0: register epilogue, scalar reduction
    (100, 20, 8192, 4, dict()),                                   # BN = 32 (K-major B planes)
    (845, 256, 65536, 40, dict()),                                # more slices than the reduction's load batch
])
def test_splitk_epilogue_cases_match_variant3(cuda, kin, nout, B, sk, kw):
    got, want = _wgrad(cuda, kin, nout, B, sk, **kw)
    assert torch.equal(got, want), float((got - want).abs().max())


def _dense_grads(cuda, m, kdim, n):
    from deepctr_b200 import engine as E
    _, _, ops = _mods()
    rng = np.random.RandomState(m + kdim + n)
    t = lambda *s: torch.tensor(rng.normal(size=s).astype(np.float32)).to(cuda)
    x, w, b = E.Var(t(m, kdim), requires_grad=True), E.Var(t(kdim, n), requires_grad=True), E.Var(t(n), requires_grad=True)
    gy = t(m, n)
    tape = E.Tape()
    with E.recording(tape):
        y = ops.dense(x, w, b, activation="relu")
    y.requires_grad = True
    E.add_grad(y, gy)
    tape.backward()
    torch.cuda.synchronize()
    return x.grad, w.grad, b.grad


@pytest.fixture
def fp32_dz(monkeypatch):
    """forces the old path: bias_act_bwd also writes the fp32 dz next to its planes"""
    _, K, _ = _mods()
    orig = K.bias_act_bwd

    def with_dz(dy, y, act, want_dz=True, want_dbias=True, m=None, n=None, want_planes=False):
        return orig(dy, y, act, want_dz=True, want_dbias=want_dbias, m=m, n=n, want_planes=want_planes)
    monkeypatch.setattr(K, "bias_act_bwd", with_dz)


@pytest.fixture
def dz_requests(monkeypatch):
    """records want_dz of every bias_act_bwd call that also writes planes"""
    _, K, _ = _mods()
    orig, seen = K.bias_act_bwd, []

    def spy(dy, y, act, want_dz=True, want_dbias=True, m=None, n=None, want_planes=False):
        if want_planes:
            seen.append(want_dz)
        return orig(dy, y, act, want_dz=want_dz, want_dbias=want_dbias, m=m, n=n, want_planes=want_planes)
    monkeypatch.setattr(K, "bias_act_bwd", spy)
    return seen


@pytest.mark.parametrize("m,kdim,n", [(8192, 845, 256), (8192, 256, 128), (8192, 128, 64)])
def test_dense_backward_without_fp32_dz(cuda, m, kdim, n, dz_requests, request):
    got = _dense_grads(cuda, m, kdim, n)
    assert dz_requests == [False]          # the fused-planes path ran and did not ask for the fp32 dz
    request.getfixturevalue("fp32_dz")
    want = _dense_grads(cuda, m, kdim, n)
    for g, w in zip(got, want):
        assert torch.equal(g, w), float((g - w).abs().max())


def test_null_operand_without_planes_raises_before_launch(cuda):
    L, K, _ = _mods()
    a = torch.randn(64, 4096, device=cuda)
    b = torch.randn(4096, 20, device=cuda)
    ap, bp = K.split_planes(a), K.split_planes(b)
    torch.cuda.synchronize()
    L.reset_launch_count()
    with pytest.raises(ValueError):
        K.gemm(None, b, trans_a=True, precision=L.GEMM_BF16X3, m=64, n=20, k=4096)
    with pytest.raises(ValueError):        # N <= 32 with B stored [K, N]: the planes cannot be used, B must be split
        K.gemm(a, None, precision=L.GEMM_BF16X3, m=64, n=20, k=4096, b_planes=bp)
    with pytest.raises(ValueError):        # the exact-fp32 mode reads no planes
        K.gemm(None, b, precision=L.GEMM_FP32, m=64, n=20, k=4096, a_planes=ap)
    assert L.launch_count() == 0
