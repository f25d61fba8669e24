"""GPU: the SENET and bilinear-interaction kernels, the layers and the FiBiNET builder.

* b2ctr_bilinear_fwd / _bwd for the three bilinear types and b2ctr_senet_fwd / _bwd against float64 over F = 2 / 26 /
  64 and E = 4 / 5 / 32 / 64, the input a window of a wider buffer, the output a strided window of a wider buffer,
  and batches that are not a multiple of a CTA's samples; both backwards are bit-identical from run to run;
* layer fixtures of the reference's own SENETLayer / BilinearInteraction (tests/golden/fibinet/, with
  model_golden_checks): through the layers, outputs and gradients in both GEMM precisions;
* with the DNN-input placement no copy wider than the dense tail touches the DNN input; a bilinear layer called eagerly
  after training is not placed;
* model fixtures (with model_golden_checks): logits and one SGD step in both GEMM precisions, placed and unplaced;
  a graph-replayed training step equals an eager one; the placement gives the results of the unplaced graph;
* the C2 shape (26 fields, E = 32, B = 65536, 13 dense features: a [65536, 20816] DNN input and a K = 20813 GEMM):
  the logits of the first and last 512 samples against the CPU oracle.
"""
import itertools

import numpy as np
import pytest
import torch

import b2_helpers as H
import model_golden_checks as C
from model_golden_checks import placement  # noqa: F401  (the placed / unplaced parameter)

pytestmark = pytest.mark.gpu

test_layer_fixture = C.gpu_layer_test("fibinet")
T = C.gpu_model_tests("fibinet")
test_model_forward_matches_reference = T.forward
test_model_sgd_step_matches_reference_gradients = T.sgd_step
test_graph_replayed_step_equals_eager = C.graph_replay_test([
    pytest.param("FiBiNET", dict(bilinear_type="interaction", dnn_hidden_units=(32, 16)), id="interaction"),
    pytest.param("FiBiNET", dict(bilinear_type="each", dnn_hidden_units=(32,)), id="each"),
    pytest.param("FiBiNET", dict(bilinear_type="all", dnn_hidden_units=()), id="all")])
test_placement_gives_the_unplaced_results = C.placement_test([
    pytest.param("FiBiNET", dict(bilinear_type="interaction", dnn_hidden_units=(32, 16)), 1e-6, 1e-7, id="interaction"),
    pytest.param("FiBiNET", dict(bilinear_type="all", dnn_hidden_units=()), 1e-6, 1e-7, id="no_dnn")])
TYPES = ("all", "each", "interaction")


def _nw(t, F):
    return 1 if t == "all" else F - 1 if t == "each" else F * (F - 1) // 2


def _ref_bilinear(x, t, W):
    """float64: x [B,F,E], W [nW,E,E] -> [B,P,E]."""
    F = x.shape[1]
    pairs = list(itertools.combinations(range(F), 2))
    i = torch.tensor([p[0] for p in pairs], device=x.device)
    j = torch.tensor([p[1] for p in pairs], device=x.device)
    k = torch.zeros_like(i) if t == "all" else i if t == "each" else torch.arange(len(pairs), device=x.device)
    return torch.einsum("bpe,peo->bpo", x[:, i, :], W[k]) * x[:, j, :]


def _ref_senet(x, W1, W2):
    a2 = torch.relu(torch.relu(x.mean(-1) @ W1) @ W2)
    return x * a2.unsqueeze(2)


def _check_bilinear(cuda, B, F, E, t, seed, tail=13):
    from deepctr_b200 import kernels as K
    rng = np.random.RandomState(seed)
    P = F * (F - 1) // 2
    buf = torch.tensor(rng.normal(0, 0.5, size=(B, F * E + tail)).astype(np.float32), device=cuda)
    xw, ldx = buf[:, :F * E], buf.stride(0)
    W = torch.tensor(rng.normal(0, 1.0 / np.sqrt(E), size=(_nw(t, F), E, E)).astype(np.float32), device=cuda)
    # output: pair p at column 3 + p*(E+2) of a [B, ld] buffer; the rest of the buffer must stay untouched
    pitch, col0 = E + 2, 3
    ld = col0 + P * pitch + 5
    out = torch.full((B, ld), 7.0, device=cuda)
    K.bilinear_fwd(xw, ldx, F, E, t, W, B, out=out, col0=col0, pitch=pitch)
    view = out[:, col0:col0 + P * pitch].reshape(B, P, pitch)
    got = view[:, :, :E]
    mask = torch.ones_like(out, dtype=torch.bool)
    mask[:, col0:col0 + P * pitch].view(B, P, pitch)[:, :, :E] = False
    assert bool((out[mask] == 7.0).all()), "the forward wrote outside its pair windows"
    g = torch.tensor(rng.normal(0, 1.0, size=(B, ld)).astype(np.float32), device=cuda)
    gv = g[:, col0:]
    dx, dW = K.bilinear_bwd(gv, ld, 0, pitch, xw, ldx, F, E, t, W, B)
    x64 = xw.double().reshape(B, F, E).requires_grad_(True)
    W64 = W.double().requires_grad_(True)
    ref = _ref_bilinear(x64, t, W64)
    g64 = g[:, col0:col0 + P * pitch].reshape(B, P, pitch)[:, :, :E].double()
    (ref * g64).sum().backward()
    H.close(got, ref.detach(), "out")
    H.close(dx.reshape(B, F, E), x64.grad, "dx")
    H.close(dW, W64.grad, "dW")
    return (gv, ld, pitch, xw, ldx, W, dx, dW)


@pytest.mark.parametrize("t", TYPES)
@pytest.mark.parametrize("E", [4, 5, 32, 64])
@pytest.mark.parametrize("F", [2, 26, 64])
def test_bilinear_kernels_match_float64(cuda, F, E, t):
    _check_bilinear(cuda, 1001 if F * E < 64 * 64 else 203, F, E, t, 7 * F + E)


@pytest.mark.parametrize("t", TYPES)
def test_bilinear_backward_is_deterministic(cuda, t):
    from deepctr_b200 import kernels as K
    gv, ld, pitch, xw, ldx, W, dx, dW = _check_bilinear(cuda, 4099, 26, 32, t, 3)
    for _ in range(2):
        dx2, dW2 = K.bilinear_bwd(gv, ld, 0, pitch, xw, ldx, 26, 32, t, W, 4099)
        assert torch.equal(dx, dx2) and torch.equal(dW, dW2)


def _check_senet(cuda, B, F, E, R, seed):
    from deepctr_b200 import kernels as K
    rng = np.random.RandomState(seed)
    buf = torch.tensor(rng.normal(0, 0.5, size=(B, F * E + 13)).astype(np.float32), device=cuda)
    xw, ldx = buf[:, :F * E], buf.stride(0)
    W1 = torch.tensor(rng.normal(0, 0.5, size=(F, R)).astype(np.float32), device=cuda)
    W2 = torch.tensor(rng.normal(0, 0.5, size=(R, F)).astype(np.float32), device=cuda)
    g = torch.tensor(rng.normal(0, 1.0, size=(B, F * E)).astype(np.float32), device=cuda)
    v, saved = K.senet_fwd(xw, ldx, F, E, W1, W2, B)
    dx, dW1, dW2 = K.senet_bwd(g, xw, ldx, F, E, W1, W2, saved, B)
    x64 = xw.double().reshape(B, F, E).requires_grad_(True)
    W164, W264 = W1.double().requires_grad_(True), W2.double().requires_grad_(True)
    ref = _ref_senet(x64, W164, W264)
    (ref * g.double().reshape(B, F, E)).sum().backward()
    H.close(v.reshape(B, F, E), ref.detach(), "V")
    H.close(dx.reshape(B, F, E), x64.grad, "dx")
    H.close(dW1, W164.grad, "dW1", 1e-4)
    H.close(dW2, W264.grad, "dW2", 1e-4)
    return (g, xw, ldx, W1, W2, saved, dx, dW1, dW2)


@pytest.mark.parametrize("E", [4, 5, 32])
@pytest.mark.parametrize("F,R", [(2, 1), (26, 8), (64, 21), (64, 64)])
def test_senet_kernels_match_float64(cuda, F, R, E):
    _check_senet(cuda, 1001, F, E, R, F + E + R)


def test_senet_backward_is_deterministic(cuda):
    from deepctr_b200 import kernels as K
    g, xw, ldx, W1, W2, saved, dx, dW1, dW2 = _check_senet(cuda, 65537, 26, 32, 8, 11)
    for _ in range(2):
        dx2, a, b = K.senet_bwd(g, xw, ldx, 26, 32, W1, W2, saved, 65537)
        assert torch.equal(dx, dx2) and torch.equal(dW1, a) and torch.equal(dW2, b)


def test_kernels_reject_unsupported_shapes(cuda):
    from deepctr_b200 import kernels as K
    x = torch.zeros((4, 65 * 4), device=cuda)
    with pytest.raises(ValueError, match="field count"):
        K.bilinear_fwd(x, 65 * 4, 65, 4, "all", torch.zeros((1, 4, 4), device=cuda), 4)
    with pytest.raises(ValueError, match="embedding_size"):
        K.bilinear_fwd(x, 65 * 4, 3, 65, "all", torch.zeros((1, 65, 65), device=cuda), 4)
    with pytest.raises(ValueError, match="field count"):
        K.senet_fwd(x, 65 * 4, 65, 4, torch.zeros((65, 2), device=cuda), torch.zeros((2, 65), device=cuda), 4)


def test_placed_step_buffer_takes_only_the_dense_tail_copy(cuda, monkeypatch):
    """With the placement, the only copy kernel that reads or writes the DNN input is the dense tail's (3 columns);
    without it, the bilinear outputs are copied by the Concat and again by combined_dnn_input."""
    from deepctr_b200 import kernels as K
    from deepctr_b200.engine import SGD
    from deepctr_b200 import inputs as I
    events = []                # ("buf", lo, hi) when a step's DNN-input buffer is made, ("copy", src, dst, cols)
    real_copy, real_buffer = K.copy2d, I.DnnInputPlacement.buffer

    def copy_spy(src, ld_src, dst, ld_dst, rows, cols, accumulate=False, src_off=0, dst_off=0):
        events.append(("copy", src.data_ptr() + 4 * src_off, dst.data_ptr() + 4 * dst_off, int(cols)))
        return real_copy(src, ld_src, dst, ld_dst, rows, cols, accumulate=accumulate, src_off=src_off,
                         dst_off=dst_off)

    def buffer_spy(self, b, device):
        v = real_buffer(self, b, device)
        st = v.data.untyped_storage()
        events.append(("buf", st.data_ptr(), st.data_ptr() + st.nbytes()))
        return v
    monkeypatch.setattr(K, "copy2d", copy_spy)
    monkeypatch.setattr(I.DnnInputPlacement, "buffer", buffer_spy)
    widths = {}
    for placed in (True, False):
        I.DNN_INPUT_PLACEMENT = placed
        try:
            model, x, y = H.criteo_model("FiBiNET", np.random.RandomState(5), dnn_hidden_units=(16,))
        finally:
            I.DNN_INPUT_PLACEMENT = True
        model.compile(SGD(0.05), "binary_crossentropy", embedding_update="sparse", step_graph="off")
        model.train_on_batch(x, y)
        del events[:]
        model.train_on_batch(x, y)
        bufs, touching = [], []
        for ev in events:
            if ev[0] == "buf":
                bufs.append(ev[1:])
            elif any(lo <= p < hi for lo, hi in bufs for p in ev[1:3]):
                touching.append(ev[3])
        assert bool(bufs) == placed
        widths[placed] = touching if placed else [ev[3] for ev in events]
    P, E_ = 45, 8
    assert widths[True] == [3], widths[True]
    assert max(widths[False]) >= 2 * P * E_, widths[False]


def test_eager_bilinear_call_after_training_is_unplaced(cuda):
    """A BilinearInteraction of a trained FiBiNET called eagerly returns its own contiguous [B,P,E] output, equal to
    the same call before the model ever ran: the DNN-input placement belongs to the model's steps only."""
    from deepctr_b200.engine import SGD
    from deepctr_b200.layers import BilinearInteraction
    model, x, y = H.criteo_model("FiBiNET", np.random.RandomState(6), dnn_hidden_units=(16,))
    layer = next(l for l in model.layers if isinstance(l, BilinearInteraction))
    assert id(layer) in model.planner.dnn_places
    model._materialize()
    gen = torch.Generator(device=cuda).manual_seed(2)
    inputs = [torch.randn((64, 1, 8), device=cuda, generator=gen) for _ in range(10)]
    before = layer(inputs).data.clone()
    model.compile(SGD(0.0), "binary_crossentropy", embedding_update="sparse", step_graph="off")
    model.train_on_batch(x, y)
    out = layer(inputs)
    assert out.owner is None and out.base is None
    assert tuple(out.data.shape) == (64, 45, 8) and out.data.is_contiguous()
    assert torch.equal(out.data, before)


def test_c2_shape_tail_rows_match_the_oracle(cuda):
    """C2: 26 fields x 1M rows, E = 32, 13 dense features, B = 65536, 'interaction' and (256, 128, 64): the DNN input is
    [65536, 20816] (5.46 GB) and the first layer is a K = 20813 split-bf16 GEMM.  The logits of the first and last 512
    samples of the full batch equal the CPU oracle's (tests/fibinet_oracle.py) on those samples, with the model's
    weights: the table rows their ids select, SENET, both stacked bilinear weights, the DNN and the output kernel."""
    import fibinet_oracle as FO
    from deepctr_b200 import engine as E, models as M
    from deepctr_b200 import feature_column as FC
    from deepctr_b200.layers import DNN, SENETLayer
    B, F, Ed, nd, V = 65536, 26, 32, 13, 1 << 20
    cols = [FC.SparseFeat("C%d" % i, V, Ed) for i in range(F)] + [FC.DenseFeat("I%d" % i, 1) for i in range(nd)]
    E.clear_session()
    model = M.FiBiNET(cols, cols, l2_reg_linear=0, l2_reg_embedding=0)
    places = model.planner.dnn_places
    pl = next(iter(places.values()))[0]
    assert (pl.width, pl.ld) == (2 * 325 * 32, 20816)
    model._materialize()
    gen = torch.Generator(device=cuda).manual_seed(1)
    for w in model.weights:       # Keras' 1e-4 embedding init would leave the pairs ~1e-9: use O(1) values
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
    bil = [None, None]
    for layer in model.layers:
        if id(layer) in places:
            bil[places[id(layer)][1]] = [w.data.cpu() for w in layer.weights]     # index 0: the SENET branch
    senet = [l for l in model.layers if isinstance(l, SENETLayer)][0]
    dnn = [l for l in model.layers if isinstance(l, DNN)][0]
    W = {"tables": tables, "linear_kernel": host("linear/linear_kernel"),
         "senet": (senet.W_1.data.cpu(), senet.W_2.data.cpu()), "bilinear": bil,
         "dnn_kernels": [k.data.cpu() for k in dnn.kernels], "dnn_biases": [b.data.cpu() for b in dnn.bias],
         "dense_kernel": host("dense/kernel")}
    with torch.no_grad():
        want, _ = FO.fibinet(xs, cols, cols, W, bilinear_type="interaction")
    want = want.numpy().reshape(-1, 1)
    np.testing.assert_allclose(full[rows], want, rtol=1e-4, atol=H.logit_tol(want))
