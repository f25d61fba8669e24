"""GPU: the FwFM and FEFM kernels, the layers and the FwFM / DeepFEFM builders.

* b2ctr_fwfm_fwd / _bwd and b2ctr_fefm_sym / _fwd / _bwd against float64 over F = 2 / 26 / 64 and E = 4 / 5 / 32 / 64,
  the input a window of a wider buffer, FEFM's scores and their gradient a column window of a wider buffer, and
  batches that are not a multiple of a CTA's samples; both backwards are bit-identical from run to run;
* the C2 shape (B = 65536, F = 26, E = 32): the input a window of the [B, 848] gather buffer, and FEFM's scores
  written behind its 845 embedding and dense columns in a [B, 1172] buffer;
* layer fixtures of the reference's own FwFMLayer / FEFMLayer (tests/golden/fefm/, with
  model_golden_checks): through the layers, outputs and gradients in both GEMM precisions;
* with the placement, the step copies no score block ;
* model fixtures (with model_golden_checks): logits and one SGD step in both GEMM precisions, placed and unplaced;
  a graph-replayed training step equals an eager one; the placement gives the results of the unplaced graph;
* C2-shaped DeepFEFM: the logits of the first and last 512 samples against the CPU oracle.
"""
import numpy as np
import pytest
import torch

import b2_helpers as H
import model_golden_checks as C
from model_golden_checks import placement  # noqa: F401  (the placed / unplaced parameter)

pytestmark = pytest.mark.gpu

test_layer_fixture = C.gpu_layer_test("fefm")
T = C.gpu_model_tests("fefm")
test_model_forward_matches_reference = T.forward
test_model_sgd_step_matches_reference_gradients = T.sgd_step
test_graph_replayed_step_equals_eager = C.graph_replay_test([
    pytest.param("FwFM", dict(dnn_hidden_units=(32, 16)), id="fwfm"),
    pytest.param("DeepFEFM", dict(dnn_hidden_units=(32, 16)), id="deepfefm"),
    pytest.param("DeepFEFM", dict(dnn_hidden_units=()), id="deepfefm_no_dnn")])
test_placement_gives_the_unplaced_results = C.placement_test([
    pytest.param("DeepFEFM", dict(dnn_hidden_units=(32, 16)), 1e-5, 1e-6, id="defaults"),
    pytest.param("DeepFEFM", dict(dnn_hidden_units=(32,), use_linear=False), 1e-5, 1e-6, id="no_linear"),
    pytest.param("DeepFEFM", dict(dnn_hidden_units=(32,), use_fefm=False), 1e-5, 1e-6, id="no_fefm_logit")])


def _ref_fwfm(x, r):
    """float64: x [B,F,E], r [F,F] -> [B,1] over the upper triangle."""
    return torch.einsum("bie,bje,ij->b", x, x, torch.triu(r, 1)).unsqueeze(1)


def _ref_fefm(x, W):
    """float64: x [B,F,E], W [P,E,E] -> [B,P], one first field at a time."""
    F = x.shape[1]
    S = W + W.transpose(1, 2)
    out, p = [], 0
    for i in range(F - 1):
        n = F - 1 - i
        t = torch.einsum("be,peo->bpo", x[:, i], S[p:p + n])
        out.append((t * x[:, i + 1:]).sum(-1))
        p += n
    return torch.cat(out, dim=1)


def _check_fwfm(cuda, B, F, E, seed, tail=13):
    from deepctr_b200 import kernels as K
    rng = np.random.RandomState(seed)
    buf = torch.tensor(rng.normal(0, 0.5, size=(B, F * E + tail)).astype(np.float32), device=cuda)
    xw, ldx = buf[:, :F * E], buf.stride(0)
    r = torch.tensor(rng.normal(0, 0.3, size=(F, F)).astype(np.float32), device=cuda)
    out = K.fwfm_fwd(xw, ldx, F, E, r, B)
    gbuf = torch.tensor(rng.normal(0, 1.0, size=(B, 3)).astype(np.float32), device=cuda)
    g = gbuf[:, 1:2]                                         # a column of a wider buffer
    dx, dR = K.fwfm_bwd(g, gbuf.stride(0), xw, ldx, F, E, r, B)
    x64 = xw.double().reshape(B, F, E).requires_grad_(True)
    r64 = r.double().requires_grad_(True)
    ref = _ref_fwfm(x64, r64)
    (ref * g.double()).sum().backward()
    H.close(out, ref.detach(), "out")
    H.close(dx.reshape(B, F, E), x64.grad, "dx")
    H.close(dR, r64.grad, "dR", 1e-4)
    assert not bool(torch.tril(dR).any()), "dR is 0 on and below the diagonal"
    return (g, gbuf.stride(0), xw, ldx, r, dx, dR)


def _check_fefm(cuda, B, F, E, seed, ldx=None, ld=None, col0=3):
    from deepctr_b200 import kernels as K
    rng = np.random.RandomState(seed)
    P = F * (F - 1) // 2
    ldx = ldx or F * E + 13
    buf = torch.tensor(rng.normal(0, 0.5, size=(B, ldx)).astype(np.float32), device=cuda)
    xw = buf[:, :F * E]
    W = torch.tensor(rng.normal(0, 1.0 / np.sqrt(E), size=(P, E, E)).astype(np.float32), device=cuda)
    S = K.fefm_sym(W)
    assert torch.equal(S, W + W.transpose(1, 2))
    # the scores go to columns [col0, col0 + P) of a [B, ld] buffer; the rest of it must stay untouched
    ld = ld or col0 + P + 5
    out = torch.full((B, ld), 7.0, device=cuda)
    K.fefm_fwd(xw, ldx, F, E, S, B, out=out, col0=col0)
    got = out[:, col0:col0 + P]
    mask = torch.ones_like(out, dtype=torch.bool)
    mask[:, col0:col0 + P] = False
    assert bool((out[mask] == 7.0).all()), "the forward wrote outside its window"
    g = torch.tensor(rng.normal(0, 1.0, size=(B, ld)).astype(np.float32), device=cuda)
    dx, dW = K.fefm_bwd(g, ld, col0, xw, ldx, F, E, S, B)
    x64 = xw.double().reshape(B, F, E).requires_grad_(True)
    W64 = W.double().requires_grad_(True)
    ref = _ref_fefm(x64, W64)
    (ref * g[:, col0:col0 + P].double()).sum().backward()
    H.close(got, ref.detach(), "out")
    H.close(dx.reshape(B, F, E), x64.grad, "dx")
    H.close(dW, W64.grad, "dW", 1e-4)
    return (g, ld, col0, xw, ldx, S, dx, dW)


@pytest.mark.parametrize("E", [4, 5, 32, 64])
@pytest.mark.parametrize("F", [2, 26, 64])
def test_fwfm_kernels_match_float64(cuda, F, E):
    _check_fwfm(cuda, 1001, F, E, 3 * F + E)


@pytest.mark.parametrize("E", [4, 5, 32, 64])
@pytest.mark.parametrize("F", [2, 26, 64])
def test_fefm_kernels_match_float64(cuda, F, E):
    _check_fefm(cuda, 1001 if F * E < 64 * 64 else 203, F, E, 5 * F + E)


def test_kernels_at_c2_shape(cuda):
    """B = 65536, F = 26, E = 32: x a window of the [B, 848] gather buffer (832 embedding + 13 dense columns, padded
    to 848); FEFM's 325 scores at column 845 of a [B, 1172] buffer, where DeepFEFM's DNN input would hold them."""
    B = 65536
    _check_fwfm(cuda, B, 26, 32, 1, tail=848 - 832)
    _check_fefm(cuda, B, 26, 32, 2, ldx=848, ld=1172, col0=845)


def test_backwards_are_deterministic(cuda):
    from deepctr_b200 import kernels as K
    g, ldg, xw, ldx, r, dx, dR = _check_fwfm(cuda, 65537, 26, 32, 7)
    for _ in range(2):
        dx2, dR2 = K.fwfm_bwd(g, ldg, xw, ldx, 26, 32, r, 65537)
        assert torch.equal(dx, dx2) and torch.equal(dR, dR2)
    g, ld, col0, xw, ldx, S, dx, dW = _check_fefm(cuda, 4099, 26, 32, 8)
    for _ in range(2):
        dx2, dW2 = K.fefm_bwd(g, ld, col0, xw, ldx, 26, 32, S, 4099)
        assert torch.equal(dx, dx2) and torch.equal(dW, dW2)


def test_kernels_reject_unsupported_shapes(cuda):
    from deepctr_b200 import kernels as K
    x = torch.zeros((4, 65 * 65), device=cuda)
    for F, E in ((65, 4), (1, 4), (3, 65)):
        with pytest.raises(ValueError, match="field count"):
            K.fwfm_fwd(x, 65 * 65, F, E, torch.zeros((F, F), device=cuda), 4)
        with pytest.raises(ValueError, match="field count"):
            K.fefm_fwd(x, 65 * 65, F, E, torch.zeros((max(1, F * (F - 1) // 2), E, E), device=cuda), 4)
    with pytest.raises(ValueError, match="does not fit"):
        K.fefm_fwd(x, 65 * 65, 4, 4, torch.zeros((6, 4, 4), device=cuda), 4, out=torch.zeros((4, 8), device=cuda),
                   col0=3)


def test_c2_shape_deepfefm_tail_rows_match_the_oracle(cuda):
    """C2: 26 fields x 1M rows, E = 32, 13 dense features, B = 65536 and the default (256, 128, 64) DNN over the
    [65536, 832 + 13 + 325] input.  The logits of the first and last 512 samples of the full batch equal the CPU
    oracle's (tests/fefm_oracle.py) on those samples, with the model's weights."""
    import fefm_oracle as FO
    from deepctr_b200 import engine as E, models as M
    from deepctr_b200 import feature_column as FC
    from deepctr_b200.layers import DNN, FEFMLayer
    B, F, Ed, nd, V = 65536, 26, 32, 13, 1 << 20
    cols = [FC.SparseFeat("C%d" % i, V, Ed) for i in range(F)] + [FC.DenseFeat("I%d" % i, 1) for i in range(nd)]
    E.clear_session()
    model = M.DeepFEFM(cols, cols, l2_reg_linear=0, l2_reg_embedding_feat=0)
    model._materialize()
    gen = torch.Generator(device=cuda).manual_seed(1)
    for w in model.weights:       # Keras' 1e-4 embedding init would leave the scores ~1e-9: use O(1) values
        if w.name.endswith("/embeddings"):
            w.data.copy_(torch.randn(w.data.shape, device=cuda, generator=gen) * (0.3 if w.shape[1] > 1 else 0.05))
    rng = np.random.RandomState(0)
    x = {"C%d" % i: rng.randint(0, V, size=B).astype(np.int32) for i in range(F)}
    x.update({"I%d" % i: rng.rand(B).astype(np.float32) for i in range(nd)})
    full = H.logits(model, x)
    assert np.isfinite(full).all()

    rows = np.r_[0:512, B - 512:B]
    wd = {w.name: w for w in model.weights}

    def host(name, ids=None):
        t = wd[name].data
        return (t[torch.as_tensor(ids, device=cuda)] if ids is not None else t).cpu()
    xs, tables = {}, {}
    for i in range(F):           # only the rows the 1024 samples use, ids renumbered into them
        uniq, inv = np.unique(x["C%d" % i][rows], return_inverse=True)
        xs["C%d" % i] = inv.astype(np.int32)
        for prefix in ("", "linear0"):
            tables["%ssparse_emb_C%d" % (prefix, i)] = host("%ssparse_emb_C%d/embeddings" % (prefix, i), uniq)
    xs.update({"I%d" % i: x["I%d" % i][rows] for i in range(nd)})
    fefm = [l for l in model.layers if isinstance(l, FEFMLayer)][0]
    dnn = [l for l in model.layers if isinstance(l, DNN)][0]
    W = {"tables": tables, "linear_kernel": host("linear/linear_kernel"),
         "fefm": [w.data.cpu() for w in fefm.weights],
         "dnn_kernels": [k.data.cpu() for k in dnn.kernels], "dnn_biases": [b.data.cpu() for b in dnn.bias],
         "dense_kernel": host("dense/kernel")}
    with torch.no_grad():
        want, _ = FO.deepfefm(xs, cols, cols, W)
    want = want.numpy().reshape(-1, 1)
    np.testing.assert_allclose(full[rows], want, rtol=1e-4, atol=H.logit_tol(want))


def test_placed_step_copies_no_score_block(cuda, monkeypatch):
    """With the placement the scores are written into the gather buffer behind the dense tail and DeepFEFM's DNN input
    is a window of it: no copy kernel moves a block of P = 45 or more columns, in the forward or the backward.  What
    remains of that width are gradient accumulations, which the unplaced step does as well: the FEFM logit's into the
    score columns and FEFM's dx into the embedding columns.  Without the placement, the concatenation copies the
    [B, 80 + 3] and [B, 45] blocks into a new buffer forward and out of its gradient again backward."""
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
            model, x, y = H.criteo_model("DeepFEFM", np.random.RandomState(5), dnn_hidden_units=(16,))
        finally:
            I.DNN_INPUT_PLACEMENT = True
        assert bool(model.planner.fefm_places) == placed
        model.compile(SGD(0.05), "binary_crossentropy", embedding_update="sparse", step_graph="off")
        model.train_on_batch(x, y)
        del calls[:]
        model.train_on_batch(x, y)
        wide[placed] = [c for c, acc in calls if c >= P and not acc]
    assert wide[True] == [], wide[True]
    assert sorted(wide[False]) == [P, P, 80 + 3, 80 + 3], wide[False]
