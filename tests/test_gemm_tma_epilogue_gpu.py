"""GPU: the persistent split-bf16 GEMM stores plain outputs through shared memory with TMA (store_acc_tma) and keeps
the register epilogue for split-K, accumulate and C that TMA cannot address.  Both epilogues apply the same fp32
operations to the same accumulator, so variant 4 must equal variant 3 (non-persistent kernel, register epilogue)
bit for bit, and must leave every element of C outside [m, n) untouched."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

SENTINEL = 7.0


def _kern():
    from deepctr_b200 import kernels as K, _lib as L
    return K, L


def _r(rng, *shape):
    return torch.tensor(rng.normal(size=shape).astype(np.float32))


def _run(cuda, m, n, k, ta, tb, ldc, col0=0, sk=1, accumulate=False, bias=True, act="relu", alpha=1.0):
    """C = act(alpha op(A) op(B) [+ C] [+ bias]) written into columns [col0, col0 + n) of an [m, ldc] buffer filled
    with SENTINEL, for variants 3 and 4; returns both buffers."""
    K, L = _kern()
    rng = np.random.RandomState(m + 7 * n + k + ldc)
    a = _r(rng, *((k, m) if ta else (m, k))).to(cuda)
    b = _r(rng, *((n, k) if tb else (k, n))).to(cuda)
    bv = _r(rng, n).to(cuda) if bias else None
    c0 = _r(rng, m, n).to(cuda)
    outs = []
    for variant in (3, 4):
        buf = torch.full((m, ldc), SENTINEL, device=cuda)
        c = buf[:, col0:col0 + n]
        if accumulate:
            c.copy_(c0)
        K.gemm(a, b, c=c, bias=bv, trans_a=ta, trans_b=tb, act=L.ACT_RELU if act == "relu" else L.ACT_NONE,
               accumulate=accumulate, alpha=alpha, split_k=sk, precision=L.GEMM_BF16X3, m=m, n=n, k=k,
               variant=variant)
        outs.append(buf)
    torch.cuda.synchronize()
    want, got = outs
    assert torch.equal(want, got), float((want - got).abs().max())
    outside = torch.ones_like(got, dtype=torch.bool)
    outside[:, col0:col0 + n] = False
    assert bool((got[outside] == SENTINEL).all())
    # and against the exact-fp32 path
    ref = torch.full((m, ldc), SENTINEL, device=cuda)
    if accumulate:
        ref[:, col0:col0 + n].copy_(c0)
    K.gemm(a, b, c=ref[:, col0:col0 + n], bias=bv, trans_a=ta, trans_b=tb,
           act=L.ACT_RELU if act == "relu" else L.ACT_NONE, accumulate=accumulate, alpha=alpha, split_k=sk,
           m=m, n=n, k=k)
    torch.testing.assert_close(got, ref, rtol=2e-4, atol=2e-3 * max(1.0, (k / 256.0) ** 0.5))
    return got


@pytest.mark.parametrize("m,n,k,ta,tb", [
    (1000, 256, 845, False, False),     # m not a multiple of 128, BN = 128, two 64-column halves
    (130, 64, 128, False, True),        # BN = 64, second warpgroup of the last tile mostly past m
    (300, 20, 200, False, False),       # BN = 32: one 32-column box per warpgroup
    (257, 40, 64, True, False),         # BN = 64 with 24 clipped columns, MN-major A
    (40000, 256, 845, False, False),    # many tiles per CTA: the staging buffers are reused across tiles
    (30000, 64, 128, False, True),
])
def test_tma_epilogue_matches_register_epilogue(cuda, m, n, k, ta, tb):
    _run(cuda, m, n, k, ta, tb, ldc=n + (-n) % 4)


@pytest.mark.parametrize("act,bias,alpha", [("relu", True, 1.0), ("none", False, 0.5), ("none", True, -2.0)])
def test_tma_epilogue_bias_act_alpha(cuda, act, bias, alpha):
    _run(cuda, 513, 128, 256, False, False, ldc=128, bias=bias, act=act, alpha=alpha)


def test_tma_epilogue_padded_ldc_leaves_pad_columns(cuda):
    """the dgrad of the first DeepFM layer: n = 845 written into a [B, 848] buffer"""
    got = _run(cuda, 4096, 845, 256, False, True, ldc=848)
    assert bool((got[:, 845:] == SENTINEL).all())


@pytest.mark.parametrize("case", ["accumulate", "split_k", "misaligned_c", "odd_ldc"])
def test_register_epilogue_fallbacks(cuda, case):
    """outputs TMA cannot or must not store take the register epilogue and still match variant 3"""
    if case == "accumulate":          # (accumulate with an activation is rejected by b2ctr_gemm)
        _run(cuda, 1000, 256, 845, False, False, ldc=256, accumulate=True, act="none", alpha=0.5)
    elif case == "split_k":
        _run(cuda, 845, 256, 8200, True, False, ldc=256, sk=8, bias=False, act="none")
    elif case == "misaligned_c":      # C starts 4 bytes into a 16-byte aligned buffer
        _run(cuda, 1000, 128, 256, False, False, ldc=132, col0=1)
    else:                             # row pitch of 130 floats is not a multiple of 16 bytes
        _run(cuda, 1000, 128, 256, False, False, ldc=130)
