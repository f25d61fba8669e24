"""GPU: the SENET and bilinear-interaction kernels, the layers and the FiBiNET builder.

* b2ctr_bilinear_fwd / _bwd for the three bilinear types and b2ctr_senet_fwd / _bwd against float64 over F = 2 / 26 /
  64 and E = 4 / 5 / 32 / 64, the input a window of a wider buffer, the output a strided window of a wider buffer,
  and batches that are not a multiple of a CTA's samples; both backwards are bit-identical from run to run;
* layer fixtures of the reference's own SENETLayer / BilinearInteraction (tests/golden/fibinet/);
* model fixtures (tests/golden/models_fibinet/): logits and one SGD step in both GEMM precisions;
* a graph-replayed training step equals an eager one; the DNN-input placement gives the results of the unplaced
  graph, and with it no copy wider than the dense tail touches the DNN input;
* the C2 shape (26 fields, E = 32, B = 65536, 13 dense features: a [65536, 20816] DNN input and a K = 20813 GEMM):
  the logits of the first and last 512 samples against the CPU oracle.
"""
import itertools

import numpy as np
import pytest
import torch

import golden_models as G
import test_fibinet_goldens as FG

pytestmark = pytest.mark.gpu
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


def _close(got, want, what, tol=2e-5):
    scale = max(float(want.abs().max()), 1e-30)
    err = float((got.double() - want).abs().max()) / scale
    assert err < tol, "%s: max error %.3e relative to max |value|" % (what, err)


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
    _close(got, ref.detach(), "out")
    _close(dx.reshape(B, F, E), x64.grad, "dx")
    _close(dW, W64.grad, "dW")
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
    _close(v.reshape(B, F, E), ref.detach(), "V")
    _close(dx.reshape(B, F, E), x64.grad, "dx")
    _close(dW1, W164.grad, "dW1", 1e-4)
    _close(dW2, W264.grad, "dW2", 1e-4)
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


@pytest.mark.parametrize("name", FG.LAYER_CASES)
def test_layer_fixture(cuda, name):
    from deepctr_b200 import kernels as K
    meta, d = FG.load_layer(name)
    x = torch.tensor(d["x"], device=cuda)
    B, F, Ed = x.shape
    ws = [torch.tensor(d["w_" + k], device=cuda) for k in FG.layer_weight_names(d)]
    dout = torch.tensor(d["dout"], device=cuda).reshape(B, -1).contiguous()
    tol = dict(rtol=1e-4, atol=1e-5)
    if meta["layer"] == "SENETLayer":
        v, saved = K.senet_fwd(x.reshape(B, -1), F * Ed, F, Ed, ws[0], ws[1], B)
        dx, dW1, dW2 = K.senet_bwd(dout, x.reshape(B, -1), F * Ed, F, Ed, ws[0], ws[1], saved, B)
        grads = [dW1, dW2]
        out = v
    else:
        t = meta["kwargs"]["bilinear_type"]
        W = torch.stack(ws)
        out = K.bilinear_fwd(x.reshape(B, -1), F * Ed, F, Ed, t, W, B)
        dx, dW = K.bilinear_bwd(dout, dout.stride(0), 0, Ed, x.reshape(B, -1), F * Ed, F, Ed, t, W, B)
        grads = list(dW)
    np.testing.assert_allclose(out.reshape(d["out"].shape).cpu().numpy(), d["out"], **tol)
    np.testing.assert_allclose(dx.reshape(B, F, Ed).cpu().numpy(), d["gx"], **tol)
    for k, gk in zip(FG.layer_weight_names(d), grads):
        np.testing.assert_allclose(gk.cpu().numpy(), d["g_" + k], err_msg=k, **tol)


# ---- model level ----------------------------------------------------------------------------------
@pytest.fixture(params=[True, False], ids=["placed", "unplaced"])
def placement(request):
    from deepctr_b200 import inputs as I
    I.DNN_INPUT_PLACEMENT = request.param
    yield request.param
    I.DNN_INPUT_PLACEMENT = True


def _model(fx):
    model = FG.build(fx)
    return model, G.assign_weights(fx, model)


@pytest.mark.usefixtures("gemm_precision", "placement")
@pytest.mark.parametrize("name", FG.MODEL_CASES)
def test_model_forward_matches_reference(cuda, name):
    from test_model_goldens_gpu import _logits, _tol
    fx = FG.Fixture(name)
    model, _ = _model(fx)
    x = fx.inputs()
    np.testing.assert_allclose(_logits(model, x), fx.logit, rtol=1e-4, atol=_tol(fx.logit))
    np.testing.assert_allclose(model.predict(x, batch_size=len(fx.y)), fx.out, rtol=1e-4, atol=_tol(fx.out))


@pytest.mark.usefixtures("gemm_precision", "placement")
@pytest.mark.parametrize("name", FG.MODEL_CASES)
def test_model_sgd_step_matches_reference_gradients(cuda, name):
    from deepctr_b200.engine import SGD
    fx = FG.Fixture(name)
    model, wm = _model(fx)
    lr = 0.5
    model.compile(SGD(lr), "binary_crossentropy", embedding_update="dense")
    loss = model.train_on_batch(fx.inputs(), fx.y)
    assert abs(loss - fx.loss) <= 2e-4 * max(1.0, abs(fx.loss)), (loss, fx.loss)
    for key, w in wm.items():
        if key not in fx.g:
            continue
        want = fx.g[key]
        got = (fx.w[key] - w.value()) / lr
        np.testing.assert_allclose(got, want, rtol=2e-3, atol=3e-4 * float(np.abs(want).max()) + 2e-6, err_msg=key)


def _criteo_model(rng, n_dense, n=512, dim=8, **kw):
    from deepctr_b200 import engine as E, models as M
    from deepctr_b200 import feature_column as FC
    cols = [FC.SparseFeat("C%d" % i, 50 + i, dim) for i in range(10)]
    cols += [FC.DenseFeat("I%d" % i, 1) for i in range(n_dense)]
    E.clear_session()
    model = M.FiBiNET(cols, cols, l2_reg_linear=0, l2_reg_embedding=0, seed=3, **kw)
    x = {"C%d" % i: rng.randint(0, 50 + i, size=n).astype(np.int32) for i in range(10)}
    x.update({"I%d" % i: rng.rand(n).astype(np.float32) for i in range(n_dense)})
    y = (rng.rand(n) < 0.3).astype(np.float32)
    return model, x, y


def _train(placed, graph, kw, steps=6, init=None):
    from deepctr_b200 import inputs as I
    from deepctr_b200.engine import SGD
    I.DNN_INPUT_PLACEMENT = placed
    try:
        model, x, y = _criteo_model(np.random.RandomState(4), 3, **kw)
    finally:
        I.DNN_INPUT_PLACEMENT = True
    assert bool(model.planner.dnn_places) == placed
    if init is None:            # Keras leaves the final Dense kernel unseeded: start every run from the same weights
        init = [w.value() for w in model.weights]
    else:
        model.set_weights(init)
    model.compile(SGD(0.05), "binary_crossentropy", embedding_update="sparse", step_graph=graph)
    losses = [model.train_on_batch(x, y) for _ in range(steps)]
    return losses, {w.name: w.value() for w in model.weights}, model.replayed_launches, init


@pytest.mark.parametrize("kw", [dict(bilinear_type="interaction", dnn_hidden_units=(32, 16)),
                                dict(bilinear_type="each", dnn_hidden_units=(32,)),
                                dict(bilinear_type="all", dnn_hidden_units=())], ids=["interaction", "each", "all"])
def test_graph_replayed_step_equals_eager(cuda, kw):
    l_graph, w_graph, replayed, init = _train(True, "auto", kw)
    l_eager, w_eager, _, _ = _train(True, "off", kw, init=init)
    assert replayed > 0, "the training step was never replayed as a CUDA graph"
    np.testing.assert_allclose(l_graph, l_eager, rtol=1e-5, atol=1e-6)
    for k, v in w_eager.items():
        np.testing.assert_allclose(w_graph[k], v, rtol=1e-4, atol=1e-6 + 1e-4 * float(np.abs(v).max()), err_msg=k)


@pytest.mark.parametrize("kw", [dict(bilinear_type="interaction", dnn_hidden_units=(32, 16)),
                                dict(bilinear_type="all", dnn_hidden_units=())], ids=["interaction", "no_dnn"])
def test_placement_gives_the_unplaced_results(cuda, kw):
    l_p, w_p, _, init = _train(True, "off", kw)
    l_u, w_u, _, _ = _train(False, "off", kw, init=init)
    np.testing.assert_allclose(l_p, l_u, rtol=1e-6, atol=0)
    for k, v in w_u.items():
        np.testing.assert_allclose(w_p[k], v, rtol=1e-6, atol=1e-7 * float(np.abs(v).max()), err_msg=k)


def test_placed_step_copies_only_the_dense_tail(cuda, monkeypatch):
    """With the placement, the only copy kernel that reads or writes the DNN input is the dense tail's (3 columns);
    without it, the bilinear outputs are copied by the Concat and again by combined_dnn_input."""
    from deepctr_b200 import kernels as K
    from deepctr_b200.engine import SGD
    from deepctr_b200 import inputs as I
    events = []                # ("buf", lo, hi) when a step's DNN-input buffer is made, ("copy", src, dst, cols)
    real_copy, real_view = K.copy2d, I.DnnInputPlacement.out_view

    def copy_spy(src, ld_src, dst, ld_dst, rows, cols, accumulate=False, src_off=0, dst_off=0):
        events.append(("copy", src.data_ptr() + 4 * src_off, dst.data_ptr() + 4 * dst_off, int(cols)))
        return real_copy(src, ld_src, dst, ld_dst, rows, cols, accumulate=accumulate, src_off=src_off,
                         dst_off=dst_off)

    def view_spy(self, k, b, device):
        v = real_view(self, k, b, device)
        st = v.untyped_storage()
        events.append(("buf", st.data_ptr(), st.data_ptr() + st.nbytes()))
        return v
    monkeypatch.setattr(K, "copy2d", copy_spy)
    monkeypatch.setattr(I.DnnInputPlacement, "out_view", view_spy)
    widths = {}
    for placed in (True, False):
        I.DNN_INPUT_PLACEMENT = placed
        try:
            model, x, y = _criteo_model(np.random.RandomState(5), 3, dnn_hidden_units=(16,))
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


def test_c2_shape_tail_rows_match_the_oracle(cuda):
    """C2: 26 fields x 1M rows, E = 32, 13 dense features, B = 65536, 'interaction' and (256, 128, 64): the DNN input is
    [65536, 20816] (5.46 GB) and the first layer is a K = 20813 split-bf16 GEMM.  The logits of the first and last 512
    samples of the full batch equal the CPU oracle's (tests/fibinet_oracle.py) on those samples, with the model's
    weights: the table rows their ids select, SENET, both stacked bilinear weights, the DNN and the output kernel."""
    import fibinet_oracle as FO
    from deepctr_b200 import engine as E, models as M
    from deepctr_b200 import feature_column as FC
    from deepctr_b200.layers import DNN, SENETLayer
    from test_model_goldens_gpu import _logits, _tol
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
    full = _logits(model, x)
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
    np.testing.assert_allclose(full[rows], want, rtol=1e-4, atol=_tol(want))
