"""CPU: PNN and its layers (InnerProductLayer, OutterProductLayer) against fixtures the reference's own layer and
builder code produced (tests/golden/generate_pnn.py):

1. the CPU restatement of tests/pnn_oracle.py (built on oracle/) reproduces every layer output, model logit,
   prediction, loss and gradient;
2. the deepctr_b200 builder creates the reference's weight set and graph (names, shapes, order, planner slots) - only
   what is reachable from the output - and has the reference's keyword defaults;
3. the reference's checks and messages, the documented kernel limits (ValueError), get_config and Reshape;
4. the placement of PNN's products in the DNN input is planned for PNN's graph, and only there.
"""
import glob
import inspect
import json
import os

import numpy as np
import pytest
import torch

import golden_models as G
from test_reference_builders_dropin import signature

HERE = os.path.dirname(os.path.abspath(__file__))
LAYERS = os.path.join(HERE, "golden", "pnn")
MODELS = os.path.join(HERE, "golden", "models_pnn")
BUILDERS_JSON = os.path.join(HERE, "golden", "reference_builders_pnn.json")
LAYER_CASES = sorted(os.path.basename(p)[:-4] for p in glob.glob(os.path.join(LAYERS, "*.npz")))
MODEL_CASES = sorted(os.path.basename(p)[:-4] for p in glob.glob(os.path.join(MODELS, "*.npz")))


def load_layer(name):
    d = np.load(os.path.join(LAYERS, name + ".npz"))
    meta = json.loads(str(d["meta"]))
    return meta, {k: d[k] for k in d.files if k != "meta"}


class Fixture(G.Fixture):
    """golden_models.Fixture read from tests/golden/models_pnn/."""

    def __init__(self, name):
        d = np.load(os.path.join(MODELS, name + ".npz"))
        self.name = name
        self.meta = json.loads(str(d["meta"]))
        self.x = {k[2:]: d[k] for k in d.files if k.startswith("x_")}
        self.y = d["y"]
        self.w = {k[2:]: d[k] for k in d.files if k.startswith("w_")}
        self.g = {k[2:]: d[k] for k in d.files if k.startswith("g_")}
        self.out, self.logit, self.loss = d["out"], d["logit"], float(d["loss"])
        self.builder, self.kwargs = self.meta["builder"], self.meta["kwargs"]
        self.task = self.meta.get("task", "binary")
        self.training = bool(self.meta.get("training"))


def pnn_builder_args(fx):
    """PNN(dnn_feature_columns, **kwargs): the one positional argument (pnn.py:18)."""
    from deepctr_b200 import feature_column as FC
    kw = dict(fx.kwargs)
    if "dnn_hidden_units" in kw:
        kw["dnn_hidden_units"] = tuple(kw["dnn_hidden_units"])
    return (G.columns(fx, "dnn", FC),), kw


def oracle_weights(fx, requires_grad=False):
    """golden_models.oracle_weights plus W['outer'], the OutterProductLayer kernel when it is on the output path."""
    W, leaves = G.oracle_weights(fx, requires_grad)
    for n in fx.layer_names("OutterProductLayer"):
        W["outer"] = torch.tensor(fx.w[n + "/kernel"], requires_grad=requires_grad)
        leaves[n + "/kernel"] = W["outer"]
    return W, leaves


def oracle_forward(fx, W):
    import pnn_oracle as PO
    from deepctr_b200 import feature_column as FC
    kw = fx.kwargs
    return PO.pnn(fx.inputs(), G.columns(fx, "dnn", FC), W, use_inner=kw.get("use_inner", True),
                  use_outter=kw.get("use_outter", False), kernel_type=kw.get("kernel_type", "mat"), task=fx.task)


def build(fx):
    from deepctr_b200 import engine as E
    from deepctr_b200 import models as M
    args, kw = pnn_builder_args(fx)
    E.clear_session()
    return M.PNN(*args, **kw)


def test_fixture_sets():
    assert len(LAYER_CASES) == 15 and len(MODEL_CASES) == 9
    assert {Fixture(n).builder for n in MODEL_CASES} == {"PNN"}
    assert {Fixture(n).task for n in MODEL_CASES} == {"binary", "regression"}
    assert {load_layer(n)[0]["layer"] for n in LAYER_CASES} == {"InnerProductLayer", "OutterProductLayer"}


def oracle_layer(meta, x, kernel):
    import pnn_oracle as PO
    kw = meta["kwargs"]
    if meta["layer"] == "InnerProductLayer":
        return PO.inner(x, kw.get("reduce_sum", True))
    return PO.outer(x, kernel, kw["kernel_type"])


@pytest.mark.parametrize("name", LAYER_CASES)
def test_oracle_matches_reference_layer(name):
    meta, d = load_layer(name)
    x = torch.tensor(d["x"], requires_grad=True)
    k = torch.tensor(d["w_kernel"], requires_grad=True) if "w_kernel" in d else None
    out = oracle_layer(meta, x, k)
    np.testing.assert_allclose(out.detach().numpy(), d["out"], rtol=1e-5, atol=1e-6)
    (out * torch.as_tensor(d["dout"])).sum().backward()
    np.testing.assert_allclose(x.grad.numpy(), d["gx"], rtol=1e-4, atol=1e-6)
    if k is not None:
        np.testing.assert_allclose(k.grad.numpy(), d["g_kernel"], rtol=1e-4, atol=1e-6)


@pytest.mark.parametrize("name", MODEL_CASES)
def test_oracle_matches_reference_model(name):
    fx = Fixture(name)
    W, leaves = oracle_weights(fx, requires_grad=True)
    logit, pred = oracle_forward(fx, W)
    np.testing.assert_allclose(logit.detach().numpy().reshape(-1, 1), fx.logit, rtol=1e-4, atol=1e-5)
    np.testing.assert_allclose(pred.detach().numpy().reshape(-1, 1), fx.out, rtol=1e-4, atol=1e-6)
    loss = G.loss_of(fx, pred)
    assert abs(float(loss.detach()) - fx.loss) <= 1e-5 * max(1.0, abs(fx.loss))
    loss.backward()
    assert set(k for k in fx.g if not G._ignored(k)) <= set(leaves)
    for key, want in fx.g.items():
        leaf = leaves[key]
        got = leaf.grad.numpy() if leaf.grad is not None else np.zeros_like(want)
        np.testing.assert_allclose(got, want, rtol=1e-4, atol=1e-4 * float(np.abs(want).max()) + 1e-7, err_msg=key)


@pytest.mark.parametrize("name", MODEL_CASES)
def test_builder_creates_the_reference_weight_set(name):
    fx = Fixture(name)
    model = build(fx)
    wm = G.weight_map(fx, model)
    assert len(wm) == len(fx.w)
    assert [w.name for w in model.weights] == list(fx.w), "weight order"
    for key, w in wm.items():
        assert w.trainable == (key in fx.g), key


@pytest.mark.parametrize("name", MODEL_CASES)
def test_builder_graph_is_the_reference_graph(name):
    with open(BUILDERS_JSON) as f:
        want = json.load(f)["signatures"][name]
    got = signature(build(Fixture(name)))
    assert want["inputs"] == got["inputs"]
    assert want["weights"] == got["weights"]
    assert want["slots"] == got["slots"] and want["fast"] == got["fast"]
    assert sorted(want["layers"]) == sorted(got["layers"])


def test_off_path_products_hold_no_weights():
    """The reference always builds and calls OutterProductLayer (and InnerProductLayer); the one a model does not
    use is off the output path, so the graph holds neither it nor its kernel."""
    for name, inner, outer in (("pnn_defaults", True, False), ("pnn_opnn_mat", False, True),
                               ("pnn_no_products", False, False), ("pnn_inner_outer_mat", True, True)):
        model = build(Fixture(name))
        kinds = {type(l).__name__ for l in model.layers}
        assert ("InnerProductLayer" in kinds) == inner, name
        assert ("OutterProductLayer" in kinds) == outer, name
        assert any(w.name.endswith("/kernel") and "outter" in w.name for w in model.weights) == outer, name


def test_reference_default_arguments_are_the_same():
    from deepctr_b200 import models as M
    with open(BUILDERS_JSON) as f:
        ref = json.load(f)["defaults"]
    assert sorted(ref) == ["PNN"]
    mine = inspect.signature(M.PNN)
    assert [k for k, _ in ref["PNN"]] == list(mine.parameters)
    for k, d in ref["PNN"]:
        assert d == repr(mine.parameters[k].default), k


def test_bad_kernel_type_raises():
    from deepctr_b200 import engine as E, models as M
    from deepctr_b200 import feature_column as FC
    from deepctr_b200.layers import OutterProductLayer
    cols = [FC.SparseFeat("C%d" % i, 30, 4) for i in range(4)]
    E.clear_session()
    with pytest.raises(ValueError) as e:
        M.PNN(cols, kernel_type="diag")
    assert str(e.value) == "kernel_type must be mat,vec or num"
    with pytest.raises(ValueError) as e:
        OutterProductLayer("diag")
    assert str(e.value) == "kernel_type must be mat,vec or num"


@pytest.mark.parametrize("nfields,dim", [(65, 4), (3, 65)])
def test_unsupported_shapes_raise(nfields, dim):
    from deepctr_b200 import engine as E
    from deepctr_b200.layers import InnerProductLayer, OutterProductLayer
    E.clear_session()
    shapes = [(None, 1, dim)] * nfields
    with pytest.raises(ValueError, match="InnerProductLayer supports 2 to 64 inputs and embedding_size 1 to 64"):
        InnerProductLayer().build(shapes)
    with pytest.raises(ValueError, match="OutterProductLayer supports 2 to 64 inputs and embedding_size 1 to 64"):
        OutterProductLayer("vec").build(shapes)


def test_layer_reference_checks_weights_and_config():
    from deepctr_b200 import engine as E
    from deepctr_b200.layers import InnerProductLayer, OutterProductLayer
    E.clear_session()
    for cls in (InnerProductLayer, OutterProductLayer):
        n = cls.__name__
        with pytest.raises(ValueError) as e:
            cls().build([(None, 1, 4)])
        assert str(e.value) == "A `%s` layer should be called on a list of at least 2 inputs" % n
        with pytest.raises(ValueError) as e:
            cls().build([(None, 1, 4), (None, 1, 8)])
        assert str(e.value).startswith("A `%s` layer requires inputs with same shapes Got different shapes: {" % n)
        with pytest.raises(ValueError) as e:
            cls().build([(None, 2, 4), (None, 2, 4)])
        assert str(e.value) == ("A `%s` layer requires inputs of a list with same shape tensor like "
                                "(None,1,embedding_size)Got different shapes: (None, 2, 4)" % n)
    E.clear_session()
    P = 6
    for kt, shape in (("mat", (5, P, 5)), ("vec", (P, 5)), ("num", (P, 1))):
        layer = OutterProductLayer(kt, seed=7)
        layer.build([(None, 1, 5)] * 4)
        assert [(w.name.split("/")[-1], w.shape) for w in layer.weights] == [("kernel", shape)]
        assert type(layer.kernel.initializer).__name__ == "GlorotUniform" and layer.kernel.initializer.seed == 7
        assert layer.compute_output_shape([(None, 1, 5)] * 4) == (None, P)
        cfg = layer.get_config()
        assert (cfg["kernel_type"], cfg["seed"]) == (kt, 7)
    inner = InnerProductLayer(reduce_sum=False)
    inner.build([(None, 1, 5)] * 4)
    assert inner.weights == []
    assert inner.compute_output_shape([(None, 1, 5)] * 4) == (None, P, 5)
    assert InnerProductLayer().compute_output_shape([(None, 1, 5)] * 4) == (None, P, 1)
    assert inner.get_config()["reduce_sum"] is False


def test_mat_kernel_fans_follow_keras():
    """glorot_uniform on the 3-D [E, P, E] kernel: Keras' fans (P*E, E*E), from engine._fans."""
    from deepctr_b200 import engine as E
    assert E._fans((5, 6, 5)) == (6 * 5, 5 * 5)


def test_reshape_layer():
    from deepctr_b200 import engine as E
    r = E.Reshape([12])
    assert r.compute_output_shape((None, 3, 4)) == (None, 12)
    assert E.Reshape((3, -1)).compute_output_shape((None, 12)) == (None, 3, 4)
    assert r.get_config()["target_shape"] == (12,)
    with pytest.raises(ValueError, match="total size of new array must be unchanged"):
        E.Reshape([5]).compute_output_shape((None, 3, 4))


def test_pnn_placement_is_planned_for_pnn_only():
    """PNN's products get their columns between the embeddings and the dense columns of the gather buffer when its DNN
    input is concat([linear_signal, products]) through combined_dnn_input; every other model keeps its row pitch."""
    from deepctr_b200 import engine as E, inputs as I, models as M
    from deepctr_b200 import feature_column as FC
    cols = [FC.SparseFeat("C%d" % i, 30, 8) for i in range(6)] + [FC.DenseFeat("I%d" % i, 1) for i in range(3)]

    def plan(model):
        p = model.planner
        return p.main_width, p.main_ld, p.pnn_cols, sorted(p.pnn_places.values())
    # 6 x 8 = 48 embedding columns + P = 15 per product + 3 dense, padded to 4
    for kw, want in ((dict(), (48, 68, 15, [0])),
                     (dict(use_inner=False, use_outter=True), (48, 68, 15, [0])),
                     (dict(use_outter=True), (48, 84, 30, [0, 15])),
                     (dict(use_outter=True, kernel_type="num"), (48, 84, 30, [0, 15])),
                     (dict(use_inner=False), (48, 52, 0, []))):
        E.clear_session()
        assert plan(M.PNN(cols, **kw)) == want, kw
    E.clear_session()
    assert plan(M.PNN(cols[:6], use_outter=True)) == (48, 80, 30, [0, 15])     # no dense features: 78 -> 80
    for builder in ("DeepFM", "NFM", "FiBiNET", "FwFM", "DeepFEFM"):
        E.clear_session()
        model = getattr(M, builder)(cols, cols)
        assert model.planner.pnn_places == {} and model.planner.pnn_cols == 0, builder
        assert model.planner.main_ld == (68 if builder == "DeepFEFM" else 52), builder
    I.DNN_INPUT_PLACEMENT = False
    try:
        E.clear_session()
        assert plan(M.PNN(cols, use_outter=True)) == (48, 52, 0, [])
    finally:
        I.DNN_INPUT_PLACEMENT = True
