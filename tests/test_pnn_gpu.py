"""GPU: the PNN product kernels, the layers and the PNN builder.

* b2ctr_pnn_inner_fwd / _bwd (inner, elementwise, vec, num) and b2ctr_pnn_outer_fwd / _bwd (mat) against float64 over
  F = 2 / 26 / 64 and E = 4 / 5 / 32 / 64, the input a window of a wider buffer, the products and their gradient a
  column window of a wider buffer, and batches that are not a multiple of a CTA's samples; the backwards are
  bit-identical from run to run; unsupported shapes are rejected;
* the C2 shape (B = 65536, F = 26, E = 32): the input a window of the [B, 848] gather buffer, the scores at column
  845 of a wider buffer;
* layer fixtures of the reference's own InnerProductLayer / OutterProductLayer (tests/golden/pnn/, with
  model_golden_checks): through the layers, outputs and gradients in both GEMM precisions;
* the placed step copies no product-sized block; the reference test's dnn_dropout=0.5 configuration trains with a
  finite loss;
* model fixtures (with model_golden_checks): logits and one SGD step in both GEMM precisions, placed and unplaced;
  a graph-replayed training step equals an eager one; the placement gives the results of the unplaced graph.
"""
import numpy as np
import pytest
import torch

import b2_helpers as H
import model_golden_checks as C
from model_golden_checks import placement  # noqa: F401  (the placed / unplaced parameter)
import pnn_oracle as PO

pytestmark = pytest.mark.gpu

test_layer_fixture = C.gpu_layer_test("pnn")
T = C.gpu_model_tests("pnn")
test_model_forward_matches_reference = T.forward
test_model_sgd_step_matches_reference_gradients = T.sgd_step
test_graph_replayed_step_equals_eager = C.graph_replay_test([
    pytest.param("PNN", dict(dnn_hidden_units=(32, 16)), id="ipnn"),
    pytest.param("PNN", dict(dnn_hidden_units=(32, 16), use_inner=False, use_outter=True), id="opnn_mat"),
    pytest.param("PNN", dict(dnn_hidden_units=(32,), use_outter=True, kernel_type="vec"), id="both_vec"),
    pytest.param("PNN", dict(dnn_hidden_units=(32,), use_inner=False, use_outter=True, kernel_type="num"),
                 id="opnn_num")])
test_placement_gives_the_unplaced_results = C.placement_test([
    pytest.param("PNN", dict(dnn_hidden_units=(32, 16)), 1e-5, 1e-6, id="ipnn"),
    pytest.param("PNN", dict(dnn_hidden_units=(32,), use_inner=False, use_outter=True), 1e-5, 1e-6, id="opnn_mat"),
    pytest.param("PNN", dict(dnn_hidden_units=(32,), use_outter=True, kernel_type="vec"), 1e-5, 1e-6, id="both_vec"),
    pytest.param("PNN", dict(dnn_hidden_units=(32,), use_outter=True, kernel_type="num"), 1e-5, 1e-6, id="both_num")])

MODES = ["inner", "elementwise", "vec", "num", "mat"]


def _kernel(rng, mode, F, E, cuda):
    P = F * (F - 1) // 2
    shape = {"vec": (P, E), "num": (P, 1), "mat": (E, P, E)}.get(mode)
    if shape is None:
        return None
    return torch.tensor(rng.normal(0, 1.0 / np.sqrt(E), size=shape).astype(np.float32), device=cuda)


def _ref(x64, mode, K64):
    """float64 [B,F,E] -> the layer's output as [B, ncols]."""
    if mode in ("inner", "elementwise"):
        return PO.inner(x64, mode == "inner").flatten(1)
    return PO.outer(x64, K64, mode)


def _fwd(mode, xw, ldx, F, E, Kw, B, out, col0):
    from deepctr_b200 import kernels as K
    if mode == "mat":
        return K.pnn_outer_fwd(xw, ldx, F, E, Kw, B, out=out, col0=col0)
    return K.pnn_inner_fwd(xw, ldx, F, E, mode, Kw, B, out=out, col0=col0)


def _bwd(mode, g, ldg, col0, xw, ldx, F, E, Kw, B):
    from deepctr_b200 import kernels as K
    if mode == "mat":
        return K.pnn_outer_bwd(g, ldg, col0, xw, ldx, F, E, Kw, B)
    return K.pnn_inner_bwd(g, ldg, col0, xw, ldx, F, E, mode, Kw, B)


def _check(cuda, mode, B, F, E, seed, ldx=None, col0=3, ld=None, chunk=4096):
    rng = np.random.RandomState(seed)
    P = F * (F - 1) // 2
    ncols = P * E if mode == "elementwise" else P
    ldx = ldx or F * E + 13
    buf = torch.tensor(rng.normal(0, 0.5, size=(B, ldx)).astype(np.float32), device=cuda)
    xw = buf[:, :F * E]
    Kw = _kernel(rng, mode, F, E, cuda)
    # the products go to columns [col0, col0 + ncols) of a [B, ld] buffer; the rest of it must stay untouched
    ld = ld or col0 + ncols + 5
    out = torch.full((B, ld), 7.0, device=cuda)
    _fwd(mode, xw, ldx, F, E, Kw, B, out, col0)
    mask = torch.ones_like(out, dtype=torch.bool)
    mask[:, col0:col0 + ncols] = False
    assert bool((out[mask] == 7.0).all()), "the forward wrote outside its window"
    g = torch.tensor(rng.normal(0, 1.0, size=(B, ld)).astype(np.float32), device=cuda)
    dx, dK = _bwd(mode, g, ld, col0, xw, ldx, F, E, Kw, B)
    K64 = Kw.double().requires_grad_(True) if Kw is not None else None
    for b0 in range(0, B, chunk):      # float64 in sample chunks; the kernel gradient accumulates over them
        sl = slice(b0, min(B, b0 + chunk))
        x64 = xw[sl].double().reshape(-1, F, E).requires_grad_(True)
        ref = _ref(x64, mode, K64)
        (ref * g[sl, col0:col0 + ncols].double()).sum().backward()
        H.close(out[sl, col0:col0 + ncols], ref.detach(), "%s out" % mode)
        H.close(dx[sl].reshape(-1, F, E), x64.grad, "%s dx" % mode)
    if K64 is not None:
        H.close(dK, K64.grad, "%s dK" % mode, 1e-4)
    else:
        assert dK is None
    return (g, ld, col0, xw, ldx, Kw, dx, dK)


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("E", [4, 5, 32, 64])
@pytest.mark.parametrize("F", [2, 26, 64])
def test_kernels_match_float64(cuda, F, E, mode):
    B = 1001 if F * E < 64 * 64 else 203
    if mode == "elementwise" and F == 64:
        B = 67
    _check(cuda, mode, B, F, E, 7 * F + E + MODES.index(mode))


@pytest.mark.parametrize("mode", ["inner", "vec", "num", "mat"])
def test_kernels_at_c2_shape(cuda, mode):
    """B = 65536, F = 26, E = 32: x a window of the [B, 848] gather buffer (832 embedding + 13 dense columns, padded
    to 848); the 325 scores at column 845 of a [B, 1172] buffer."""
    _check(cuda, mode, 65536, 26, 32, 2, ldx=848, ld=1172, col0=845)


@pytest.mark.parametrize("mode", MODES)
def test_backwards_are_deterministic(cuda, mode):
    B = 4099
    g, ld, col0, xw, ldx, Kw, dx, dK = _check(cuda, mode, B, 26, 32, 8)
    for _ in range(2):
        dx2, dK2 = _bwd(mode, g, ld, col0, xw, ldx, 26, 32, Kw, B)
        assert torch.equal(dx, dx2)
        assert (dK is None and dK2 is None) or torch.equal(dK, dK2)


def test_kernels_reject_unsupported_shapes(cuda):
    from deepctr_b200 import kernels as K
    x = torch.zeros((4, 65 * 65), device=cuda)
    for F, E in ((65, 4), (1, 4), (3, 65)):
        P = max(1, F * (F - 1) // 2)
        with pytest.raises(ValueError, match="field count"):
            K.pnn_inner_fwd(x, 65 * 65, F, E, "inner", None, 4, out=torch.zeros((4, P), device=cuda))
        with pytest.raises(ValueError, match="field count"):
            K.pnn_outer_fwd(x, 65 * 65, F, E, torch.zeros((E, P, E), device=cuda), 4,
                            out=torch.zeros((4, P), device=cuda))
    with pytest.raises(ValueError, match="does not fit"):
        K.pnn_inner_fwd(x, 65 * 65, 4, 4, "num", torch.zeros((6, 1), device=cuda), 4,
                        out=torch.zeros((4, 8), device=cuda), col0=3)
    with pytest.raises(ValueError, match="does not fit"):
        K.pnn_outer_fwd(x, 65 * 65, 4, 4, torch.zeros((4, 6, 4), device=cuda), 4, out=torch.zeros((4, 8), device=cuda),
                        col0=3)


def test_reference_test_configuration_trains_with_dropout(cuda):
    """The reference's tests/models/PNN_test.py configuration: dnn_hidden_units=[4, 4], dnn_dropout=0.5, each of the
    use_inner / use_outter combinations; a few steps of training give finite losses."""
    from deepctr_b200.engine import SGD
    for use_inner, use_outter in ((True, True), (True, False), (False, True), (False, False)):
        model, x, y = H.criteo_model("PNN", np.random.RandomState(6), dnn_hidden_units=[4, 4], dnn_dropout=0.5,
                                     use_inner=use_inner, use_outter=use_outter)
        model.compile(SGD(0.05), "binary_crossentropy", embedding_update="sparse")
        losses = [model.train_on_batch(x, y) for _ in range(3)]
        assert np.isfinite(losses).all(), (use_inner, use_outter, losses)


def test_placed_step_copies_no_product_block(cuda, monkeypatch):
    """With the placement the products are written into the gather buffer behind the embeddings and PNN's DNN input
    is a window of it: no copy kernel moves a block of P = 45 or more columns, forward or backward (gradient
    accumulations aside: the products' dx into the embedding columns).  Without it, the two concatenations copy the
    [B, 80], [B, 45] and [B, 80 + 45] blocks into new buffers forward and out of their gradients backward."""
    from deepctr_b200 import kernels as K
    from deepctr_b200 import inputs as I
    from deepctr_b200.engine import SGD
    calls = []
    real_copy = K.copy2d

    def copy_spy(src, ld_src, dst, ld_dst, rows, cols, accumulate=False, src_off=0, dst_off=0):
        calls.append((int(cols), bool(accumulate)))
        return real_copy(src, ld_src, dst, ld_dst, rows, cols, accumulate=accumulate, src_off=src_off,
                         dst_off=dst_off)
    monkeypatch.setattr(K, "copy2d", copy_spy)
    P = 45
    wide = {}
    for placed in (True, False):
        I.DNN_INPUT_PLACEMENT = placed
        try:
            model, x, y = H.criteo_model("PNN", np.random.RandomState(5), dnn_hidden_units=(16,))
        finally:
            I.DNN_INPUT_PLACEMENT = True
        assert bool(model.planner.pnn_places) == placed
        model.compile(SGD(0.05), "binary_crossentropy", embedding_update="sparse", step_graph="off")
        model.train_on_batch(x, y)
        del calls[:]
        model.train_on_batch(x, y)
        wide[placed] = [c for c, acc in calls if c >= P and not acc]
    assert wide[True] == [], wide[True]
    assert P in wide[False] and 80 + P in wide[False], wide[False]
