"""GPU: the Bi-Interaction and fused AFM kernels, the layers and the NFM / AFM builders.

* layer fixtures of the reference's own AFMLayer / BiInteractionPooling (tests/golden/pairwise/, with
  model_golden_checks): through the layers, outputs and gradients in both GEMM precisions;
* b2ctr_afm_fwd / _bwd and b2ctr_bi_interaction_fwd / _bwd against a float64 torch restatement over F = 2 / 26 / 64,
  E = 4 / 32, A = 1 / 8, an input that is a window of a wider buffer (ldx > F*E) and batches that are not a multiple
  of the CTA's samples; the AFM backward is bit-identical from run to run;
* 'sparse' embedding updates train AFM ;
* model fixtures (with model_golden_checks): logits and one SGD step in both GEMM precisions; a graph-replayed
  training step equals an eager one;
* the C2 shape (26 fields, E = 32, A = 8, B = 65536).
"""
import numpy as np
import pytest
import torch

import b2_helpers as H
import model_golden_checks as C

pytestmark = pytest.mark.gpu

test_layer_fixture = C.gpu_layer_test("pairwise")
T = C.gpu_model_tests("pairwise")
test_model_forward_matches_reference = T.forward
test_model_sgd_step_matches_reference_gradients = T.sgd_step
test_graph_replayed_step_equals_eager = C.graph_replay_test([("NFM", dict(dnn_hidden_units=(32, 16))),
                                                          ("AFM", dict(n_dense=0, attention_factor=8)),
                                                          ("AFM", dict(n_dense=0, use_attention=False))])


def _ref_afm(x, W, b, h):
    """float64 restatement: att [B,E] of AFMLayer (layers/interaction.py:126-141)."""
    B, F, E = x.shape
    i, j = torch.triu_indices(F, F, 1, device=x.device)
    prod = x[:, i, :] * x[:, j, :]                                   # [B,P,E]
    s = torch.relu(prod @ W + b) @ h.reshape(-1, 1)                   # [B,P,1]
    return (torch.softmax(s, dim=1) * prod).sum(dim=1)


def _ref_bi(x):
    return 0.5 * (x.sum(dim=1) ** 2 - (x * x).sum(dim=1))


def _window(cuda, B, F, E, tail, rng):
    """x [B,F,E] as the leading window of a [B, F*E + tail] buffer (the gather buffer with its dense tail)."""
    buf = torch.tensor(rng.normal(0, 0.5, size=(B, F * E + tail)).astype(np.float32), device=cuda)
    return buf, buf[:, :F * E], buf.stride(0)


def _afm_weights(cuda, E, A, rng):
    W = torch.tensor(rng.normal(0, 1.0 / np.sqrt(E), size=(E, A)).astype(np.float32), device=cuda)
    b = torch.tensor(rng.normal(0, 0.1, size=(A,)).astype(np.float32), device=cuda)
    h = torch.tensor(rng.normal(0, 1.0, size=(A,)).astype(np.float32), device=cuda)
    return W, b, h


def _check_afm(cuda, B, F, E, A, tail, seed):
    from deepctr_b200 import kernels as K
    rng = np.random.RandomState(seed)
    buf, xw, ld = _window(cuda, B, F, E, tail, rng)
    tail_before = buf[:, F * E:].clone()
    W, b, h = _afm_weights(cuda, E, A, rng)
    g = torch.tensor(rng.normal(0, 1.0, size=(B, E)).astype(np.float32), device=cuda)
    att, state = K.afm_fwd(xw, ld, F, E, W, b, h, B)
    dx, dW, db, dh = K.afm_bwd(g, xw, ld, F, E, W, b, h, state, att, B)
    x64 = xw.double().reshape(B, F, E).requires_grad_(True)
    W64, b64, h64 = (t.double().requires_grad_(True) for t in (W, b, h))
    ref = _ref_afm(x64, W64, b64, h64)
    (ref * g.double()).sum().backward()
    H.close(att, ref.detach(), "att")
    H.close(dx.reshape(B, F, E), x64.grad, "dx")
    # floor: with F = 2 the softmax is exactly 1, ds = 0 and the weight gradients vanish in float64, while fp32
    # keeps the rounding of <g, prod> - <g, att> (two summation orders of the same sum)
    H.close(dW, W64.grad, "dW", floor=1e-3 * B)
    H.close(db, b64.grad, "dbias", floor=1e-3 * B)
    H.close(dh, h64.grad, "dh", floor=1e-3 * B)
    # state: max and sum of the softmax of the scores
    assert torch.isfinite(state).all() and bool((state[:, 1] >= 1.0 - 1e-6).all())
    assert torch.equal(buf[:, F * E:], tail_before)     # the dense tail behind the window is never written
    return buf, (xw, ld, W, b, h, g, state, att, dx, dW, db, dh)


@pytest.mark.parametrize("F", [2, 26, 64])
@pytest.mark.parametrize("E,A", [(4, 1), (4, 8), (32, 1), (32, 8)])
def test_afm_kernels_match_float64(cuda, F, E, A):
    _check_afm(cuda, 1001, F, E, A, 13, 100 + F + E + A)


@pytest.mark.parametrize("E,A", [(5, 3), (12, 16), (20, 6)])
def test_afm_kernels_padded_shapes(cuda, E, A):
    """E and A that are not the kernel's template sizes (padded with zero weights)."""
    _check_afm(cuda, 77, 9, E, A, 3, 7 + E + A)


def test_afm_backward_is_deterministic(cuda):
    from deepctr_b200 import kernels as K
    _, (xw, ld, W, b, h, g, state, att, dx, dW, db, dh) = _check_afm(cuda, 4099, 26, 32, 8, 13, 5)
    for _ in range(2):
        dx2, dW2, db2, dh2 = K.afm_bwd(g, xw, ld, 26, 32, W, b, h, state, att, 4099)
        assert torch.equal(dx, dx2) and torch.equal(dW, dW2) and torch.equal(db, db2) and torch.equal(dh, dh2)


@pytest.mark.parametrize("F,E", [(2, 4), (26, 32), (64, 4), (7, 40)])
def test_bi_interaction_kernels_match_float64(cuda, F, E):
    from deepctr_b200 import kernels as K
    rng = np.random.RandomState(F * E)
    B = 999
    buf, xw, ld = _window(cuda, B, F, E, 13, rng)
    tail = buf[:, F * E:].clone()
    g = torch.tensor(rng.normal(0, 1.0, size=(B, E)).astype(np.float32), device=cuda)
    out = K.bi_interaction_fwd(xw, ld, F, E, B)
    dx = K.bi_interaction_bwd(xw, ld, F, E, g, B)
    x64 = xw.double().reshape(B, F, E).requires_grad_(True)
    ref = _ref_bi(x64)
    (ref * g.double()).sum().backward()
    torch.testing.assert_close(out.double(), ref.detach(), rtol=1e-5, atol=1e-5)
    torch.testing.assert_close(dx.double().reshape(B, F, E), x64.grad, rtol=1e-5, atol=1e-5)
    assert torch.equal(buf[:, F * E:], tail)


def test_afm_kernel_rejects_unsupported_shapes(cuda):
    from deepctr_b200 import kernels as K
    x = torch.zeros((4, 65 * 4), device=cuda)
    W, b, h = torch.zeros((4, 2), device=cuda), torch.zeros(2, device=cuda), torch.zeros(2, device=cuda)
    with pytest.raises(ValueError, match="field count"):
        K.afm_fwd(x, 65 * 4, 65, 4, W, b, h, 4)


def test_afm_sparse_update_trains(cuda):
    """AFM's dx feeds the fused scatter-update: with l2 = 0, 'sparse' SGD equals 'dense' SGD."""
    from deepctr_b200.engine import SGD
    res, init = [], None
    for mode in ("sparse", "dense"):
        model, x, y = H.criteo_model("AFM", np.random.RandomState(9), n_dense=0, attention_factor=4, l2_reg_att=0)
        if init is None:
            init = [w.value() for w in model.weights]
        else:
            model.set_weights(init)
        model.compile(SGD(0.1), "binary_crossentropy", embedding_update=mode)
        losses = [model.train_on_batch(x, y) for _ in range(8)]
        res.append((losses, {w.name: w.value() for w in model.weights}))
    (ls, ws), (ld, wd) = res
    assert ls[-1] < ls[0]
    np.testing.assert_allclose(ls, ld, rtol=1e-4)
    for k, v in wd.items():
        np.testing.assert_allclose(ws[k], v, rtol=1e-3, atol=1e-3 * float(np.abs(v).max()) + 1e-7, err_msg=k)


def test_afm_c2_shape(cuda):
    """26 fields, E = 32, A = 8, B = 65536: att / dx on a random subset of rows, the weight gradients over the whole
    batch, against float64 (computed on the device in chunks)."""
    from deepctr_b200 import kernels as K
    B, F, E, A = 65536, 26, 32, 8
    rng = np.random.RandomState(2026)
    gen = torch.Generator(device=cuda).manual_seed(7)
    ld = F * E + 13 + 3
    buf = torch.randn((B, ld), device=cuda, generator=gen) * 0.3
    xw = buf[:, :F * E]
    W, b, h = _afm_weights(cuda, E, A, rng)
    g = torch.randn((B, E), device=cuda, generator=gen) * (1.0 / B)
    att, state = K.afm_fwd(xw, ld, F, E, W, b, h, B)
    dx, dW, db, dh = K.afm_bwd(g, xw, ld, F, E, W, b, h, state, att, B)
    W64, b64, h64 = (t.double().requires_grad_(True) for t in (W, b, h))
    rows = torch.tensor(np.sort(rng.choice(B, 512, replace=False)), device=cuda)
    for lo in range(0, B, 8192):
        x64 = xw[lo:lo + 8192].double().reshape(-1, F, E).requires_grad_(lo == 0 or True)
        ref = _ref_afm(x64, W64, b64, h64)
        (ref * g[lo:lo + 8192].double()).sum().backward()
        sel = rows[(rows >= lo) & (rows < lo + 8192)] - lo
        if sel.numel():
            torch.testing.assert_close(att[lo + sel].double(), ref.detach()[sel], rtol=1e-4, atol=1e-5)
            gsel = x64.grad[sel]
            scale = float(gsel.abs().max())
            torch.testing.assert_close(dx[lo + sel].double().reshape(-1, F, E), gsel, rtol=1e-4, atol=1e-5 * scale)
    # sums over 65536 x 325 terms of both signs: checked against their largest element
    for got, want in ((dW, W64.grad), (db, b64.grad), (dh, h64.grad)):
        torch.testing.assert_close(got.double(), want, rtol=1e-4, atol=1e-4 * float(want.abs().max()))
