"""The fused uniform gather's extra outputs and their use downstream:
  * the bf16 hi/lo planes of x[:, :F*E + nd] equal b2ctr_split_planes(x) bit for bit (pad columns and rows zero);
  * the stored FM sum vector S equals a float64 sum within fp32 rounding, and bit for bit an fp32 restatement of
    the order both the gather and the scatter use: ascending f per lane slot, then the xor tree over LPR .. 16;
  * the scatter reading S forms dX + dfm (S - x) as float64 does (STORE_GRADS, unique ids);
  * DeepFM steps with the planes fusion learned give the losses and weights of steps without it."""
import numpy as np
import pytest
import torch

import b2_helpers as H

pytestmark = pytest.mark.gpu


def _setup(cuda, B, F, E, nd, V=5000, seed=0, bad=True):
    from deepctr_b200 import kernels as K
    gen = torch.Generator(device=cuda).manual_seed(seed)
    tabs = [torch.randn((V, E), device=cuda, generator=gen) for _ in range(F)]
    ids = torch.randint(0, V, (B, F), device=cuda, generator=gen, dtype=torch.int32)
    if bad:
        ids[0, 0] = -1
        ids[B - 1, F - 1] = V + 3
    kd = F * E + nd
    ldx = (kd + 3) // 4 * 4 + 4
    dense = torch.randn((B, nd), device=cuda, generator=gen) if nd else None
    x = torch.full((B, ldx), float("nan"), device=cuda)
    fm = torch.empty((B,), device=cuda)
    fm_mask = sum(1 << f for f in range(F) if f % 5 != 3)
    feats = [K.make_feature(tabs[f], ids[:, f:f + 1], x, out_col=f * E, out_ld=ldx, vocab=V) for f in range(F)]
    plan = K.UniformPlan(feats, None, dense, x, None, fm, fm_mask)
    plan.g.x_cols = ldx
    return K, plan, tabs, ids, x, kd, fm_mask


@pytest.mark.parametrize("B,F,E,nd", [(65536, 26, 32, 13), (1000, 26, 4, 13), (777, 10, 8, 0), (300, 7, 16, 5),
                                      (513, 5, 64, 0), (256, 3, 32, 1)])
def test_gather_planes_equal_split_planes(cuda, B, F, E, nd):
    K, plan, tabs, ids, x, kd, _ = _setup(cuda, B, F, E, nd)
    planes = plan.set_planes(kd)
    planes.fill_(0xA5)                     # every byte, pads included, must be written
    K.embed_gather_uniform_fwd(plan, B)
    want = K.split_planes(x[:, :kd])
    torch.cuda.synchronize()
    assert planes.shape == want.shape
    pitch = 64 if kd <= 64 else (kd + 127) // 128 * 128
    n = 2 * ((B + 255) // 256 * 256) * pitch * 2            # hi then lo; b2ctr_planes_bytes adds unused slack
    assert torch.equal(planes[:n], want[:n])
    assert K.embed_oob_count() == 2


def _s_fp32_order(rows, sel, E):
    """S as the kernels sum it: lane (slot, chunk) adds features slot, slot + RPI, ... in ascending order, then
    s += shfl_xor(s, o) for o = LPR, 2 LPR, .., 16.  rows: [B, F, E] fp32 numpy (zero rows for bad ids)."""
    B, F, _ = rows.shape
    LPR = E // 4
    RPI = 32 // LPR
    part = np.zeros((B, RPI, E), dtype=np.float32)
    for f in range(F):
        if sel[f]:
            part[:, f % RPI, :] = (part[:, f % RPI, :] + rows[:, f, :]).astype(np.float32)
    o = 1
    while o < RPI:                         # lane offset o * LPR pairs slot s with slot s ^ o
        part = (part + part[:, np.arange(RPI) ^ o, :]).astype(np.float32)
        o <<= 1
    return part[:, 0, :]


@pytest.mark.parametrize("B,F,E", [(65536, 26, 32), (1000, 26, 4), (777, 10, 8), (300, 7, 16), (513, 5, 64)])
def test_gather_fm_sum(cuda, B, F, E):
    K, plan, tabs, ids, x, kd, fm_mask = _setup(cuda, B, F, E, 0)
    K.embed_gather_uniform_fwd(plan, B)
    S = plan.fm_sum.cpu().numpy()
    rows = x[:, :F * E].reshape(B, F, E).cpu().numpy()
    sel = [(fm_mask >> f) & 1 == 1 for f in range(F)]
    assert np.array_equal(S, _s_fp32_order(rows, sel, E))
    want = rows.astype(np.float64)[:, sel, :].sum(1)
    bound = np.abs(rows.astype(np.float64))[:, sel, :].sum(1) * F * 2.0 ** -24 + 1e-30
    assert (np.abs(S - want) <= bound).all()
    assert K.embed_oob_count() == 2


@pytest.mark.parametrize("E", [8, 32])
def test_scatter_with_stored_s_matches_float64(cuda, E):
    from deepctr_b200 import _lib as L
    B, F = 4096, 26
    K, plan, tabs, ids, x, kd, fm_mask = _setup(cuda, B, F, E, 0, bad=False)
    K.embed_gather_uniform_fwd(plan, B)
    gen = torch.Generator(device=cuda).manual_seed(7)
    dx = torch.randn((B, x.shape[1]), device=cuda, generator=gen)
    dfm = torch.randn((B,), device=cuda, generator=gen)
    # unique ids: row b * F + f of one gradient buffer per (sample, feature)
    grows = torch.full((B * F, E), float("nan"), device=cuda)
    pos = torch.arange(B * F, device=cuda, dtype=torch.int32).reshape(B, F)
    feats = [K.make_feature(grows, pos[:, f:f + 1], x, out_col=f * E, out_ld=x.shape[1], vocab=B * F)
             for f in range(F)]
    bplan = K.UniformPlan(feats, None, None, x, None, None, fm_mask)
    bplan.g.x_cols = x.shape[1]
    bplan.g.flags = L.UNIFORM_STORE_GRADS
    K.embed_scatter_uniform_bwd(bplan, dx, dfm, None, 0.5, 1.0, B, fm_sum=plan.fm_sum)
    xr = x[:, :F * E].reshape(B, F, E).double()
    sel = torch.tensor([(fm_mask >> f) & 1 == 1 for f in range(F)], device=cuda)
    S = (xr * sel[None, :, None]).sum(1, keepdim=True)
    want = dx[:, :F * E].reshape(B, F, E).double() + dfm.double()[:, None, None] * (S - xr) * sel[None, :, None]
    want = 0.5 * want
    got = grows.reshape(B, F, E).double()
    bound = 0.5 * (dx[:, :F * E].reshape(B, F, E).double().abs()
                   + dfm.double().abs()[:, None, None] * ((xr.abs() * sel[None, :, None]).sum(1, keepdim=True)
                                                          + xr.abs())) * (F + 4) * 2.0 ** -24 + 1e-30
    assert bool(((got - want).abs() <= bound).all())
    # the scatter reads the stored S rather than re-summing x: a shifted S shifts every FM field's row by 0.5 dfm
    K.embed_scatter_uniform_bwd(bplan, dx, dfm, None, 0.5, 1.0, B, fm_sum=plan.fm_sum + 1.0)
    shifted = grows.reshape(B, F, E).double()
    step = 0.5 * dfm.double()[:, None, None] * sel[None, :, None]
    assert bool(((shifted - got - step).abs() <= 2 * bound + 1e-6 * step.abs()).all())
    assert bool((shifted[:, ~sel] == got[:, ~sel]).all())


@pytest.mark.parametrize("prec", ["bf16x3", "fp32"])
def test_deepfm_steps_same_with_and_without_gather_planes(cuda, prec, monkeypatch):
    from deepctr_b200 import ops
    from deepctr_b200.engine import SGD
    from deepctr_b200.models import DeepFM
    from deepctr_b200.inputs import EmbeddingPlanner
    ops.set_gemm_precision(prec)
    try:
        res = []
        for fused in (True, False):
            rng = np.random.RandomState(3)
            cols, x, y = H.criteo_like(rng, 512, n_sparse=8, n_dense=3, dim=16)
            model = DeepFM(cols, cols, dnn_hidden_units=(64, 32), l2_reg_linear=0, l2_reg_embedding=0)
            H.randomize_weights(model, rng)
            model.compile(SGD(0.05), "binary_crossentropy", embedding_update="sparse")
            if not fused:
                monkeypatch.setattr(EmbeddingPlanner, "lookup_planes", lambda self, v, t2: None)
            losses, used = [], 0
            for _ in range(4):
                losses.append(model.train_on_batch(x, y))
                used += model.planner.planes_result is not None
            assert used == ((3 if prec == "bf16x3" else 0) if fused else 0)
            res.append((losses, H.flat_params(H.oracle_weights(model))))
            monkeypatch.undo()
        (l1, w1), (l2, w2) = res
        # the only run-to-run difference is the fp32 atomics of the embedding row update
        np.testing.assert_allclose(l1, l2, rtol=1e-5)
        for k in w1:
            np.testing.assert_allclose(w1[k].numpy(), w2[k].numpy(), rtol=1e-4, atol=1e-6, err_msg=k)
    finally:
        ops.set_gemm_precision("bf16x3")
