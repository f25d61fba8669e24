"""CPU: FiBiNET and its layers (SENETLayer, BilinearInteraction) against fixtures the reference's own layer and
builder code produced (tests/golden/generate_fibinet.py):

1. the CPU restatement of tests/fibinet_oracle.py (built on oracle/) reproduces every layer output, model logit,
   prediction, loss and gradient;
2. the deepctr_b200 builder creates the reference's weight set and graph (names, shapes, order, planner slots), and
   has the reference's keyword defaults;
3. the documented shape limits of the SENET / bilinear kernels raise ValueError, an unknown bilinear_type raises
   NotImplementedError;
4. the DNN-input placement is planned for FiBiNET's graph, and only there.
"""
import glob
import inspect
import json
import os
import re

import numpy as np
import pytest
import torch

import golden_models as G
from test_reference_builders_dropin import signature, builder_args

HERE = os.path.dirname(os.path.abspath(__file__))
LAYERS = os.path.join(HERE, "golden", "fibinet")
MODELS = os.path.join(HERE, "golden", "models_fibinet")
BUILDERS_JSON = os.path.join(HERE, "golden", "reference_builders_fibinet.json")
LAYER_CASES = sorted(os.path.basename(p)[:-4] for p in glob.glob(os.path.join(LAYERS, "*.npz")))
MODEL_CASES = sorted(os.path.basename(p)[:-4] for p in glob.glob(os.path.join(MODELS, "*.npz")))


def load_layer(name):
    d = np.load(os.path.join(LAYERS, name + ".npz"))
    meta = json.loads(str(d["meta"]))
    return meta, {k: d[k] for k in d.files if k != "meta"}


def layer_weight_names(d):
    """weight names of a layer fixture, in the layer's order (the npz keeps insertion order)."""
    return [k[2:] for k in d if k.startswith("w_")]


class Fixture(G.Fixture):
    """golden_models.Fixture read from tests/golden/models_fibinet/."""

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


def _creation_order(name):
    m = re.search(r"_(\d+)$", name)
    return int(m.group(1)) if m else 0


def oracle_weights(fx, requires_grad=False):
    """golden_models.oracle_weights plus the SENET weights and the two bilinear layers' weights (SENET branch
    first: the layer created first)."""
    W, leaves = G.oracle_weights(fx, requires_grad)

    def t(key):
        v = torch.tensor(fx.w[key], requires_grad=requires_grad and key in fx.g)
        leaves[key] = v
        return v
    senet = fx.layer_names("SENETLayer")[0]
    W["senet"] = (t(senet + "/W_1"), t(senet + "/W_2"))
    W["bilinear"] = [[t(k) for k in fx.w if k.startswith(name + "/bilinear_weight")]
                     for name in sorted(fx.layer_names("BilinearInteraction"), key=_creation_order)]
    W.setdefault("dnn_kernels", [])
    W.setdefault("dnn_biases", [])
    return W, leaves


def oracle_forward(fx, W):
    import fibinet_oracle as FO
    from deepctr_b200 import feature_column as FC
    lin, dnn = G.columns(fx, "linear", FC), G.columns(fx, "dnn", FC)
    return FO.fibinet(fx.inputs(), lin, dnn, W, bilinear_type=fx.kwargs.get("bilinear_type", "interaction"),
                      task=fx.task)


def build(fx):
    from deepctr_b200 import engine as E
    from deepctr_b200 import models as M
    args, kw = builder_args(fx)
    E.clear_session()
    return getattr(M, fx.builder)(*args, **kw)


def test_fixture_sets():
    assert len(LAYER_CASES) == 12 and len(MODEL_CASES) == 5
    assert set(Fixture(n).builder for n in MODEL_CASES) == {"FiBiNET"}
    assert {Fixture(n).kwargs["bilinear_type"] for n in MODEL_CASES} == {"all", "each", "interaction"}


@pytest.mark.parametrize("name", LAYER_CASES)
def test_oracle_matches_reference_layer(name):
    import fibinet_oracle as FO
    meta, d = load_layer(name)
    x = torch.tensor(d["x"], requires_grad=True)
    ws = [torch.tensor(d["w_" + k], requires_grad=True) for k in layer_weight_names(d)]
    if meta["layer"] == "SENETLayer":
        out = FO.senet(x, *ws)
    else:
        out = FO.bilinear(x, meta["kwargs"]["bilinear_type"], ws)
    np.testing.assert_allclose(out.detach().numpy(), d["out"], rtol=1e-5, atol=1e-6)
    (out * torch.as_tensor(d["dout"])).sum().backward()
    np.testing.assert_allclose(x.grad.numpy(), d["gx"], rtol=1e-4, atol=1e-6)
    for k, v in zip(layer_weight_names(d), ws):
        np.testing.assert_allclose(v.grad.numpy(), d["g_" + k], rtol=1e-4, atol=1e-6, err_msg=k)


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
        if G._ignored(key):
            assert not np.any(want), key
            continue
        leaf = leaves[key]
        got = leaf.grad.numpy() if leaf.grad is not None else np.zeros_like(want)
        np.testing.assert_allclose(got, want, rtol=1e-4, atol=1e-4 * float(np.abs(want).max()) + 1e-7, err_msg=key)


@pytest.mark.parametrize("name", MODEL_CASES)
def test_builder_creates_the_reference_weight_set(name):
    fx = Fixture(name)
    model = build(fx)
    wm = G.weight_map(fx, model)
    assert len(wm) == len([k for k in fx.w if not G._ignored(k)])
    assert [w.name for w in model.weights if not G._ignored(w.name)] == \
        [k for k in fx.w if not G._ignored(k)], "weight order"
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


def test_reference_default_arguments_are_the_same():
    from deepctr_b200 import models as M
    with open(BUILDERS_JSON) as f:
        ref = json.load(f)["defaults"]
    assert sorted(ref) == ["FiBiNET"]
    mine = inspect.signature(M.FiBiNET)
    assert [k for k, _ in ref["FiBiNET"]] == list(mine.parameters)
    for k, d in ref["FiBiNET"]:
        assert d == repr(mine.parameters[k].default), k


@pytest.mark.parametrize("nfields,dim", [(65, 4), (3, 65)])
def test_bilinear_unsupported_shapes_raise(nfields, dim):
    from deepctr_b200 import engine as E
    from deepctr_b200.layers import BilinearInteraction
    E.clear_session()
    with pytest.raises(ValueError, match="BilinearInteraction supports"):
        BilinearInteraction(bilinear_type="all").build([(None, 1, dim)] * nfields)


@pytest.mark.parametrize("nfields,ratio", [(65, 3), (4, 0.05)])
def test_senet_unsupported_shapes_raise(nfields, ratio):
    from deepctr_b200 import engine as E
    from deepctr_b200.layers import SENETLayer
    E.clear_session()
    with pytest.raises(ValueError, match="SENETLayer supports"):
        SENETLayer(reduction_ratio=ratio).build([(None, 1, 4)] * nfields)


def test_unknown_bilinear_type_raises():
    from deepctr_b200 import engine as E
    from deepctr_b200.layers import BilinearInteraction
    E.clear_session()
    with pytest.raises(NotImplementedError):
        BilinearInteraction(bilinear_type="outer").build([(None, 1, 4)] * 3)


def test_layer_reference_checks_weights_and_config():
    from deepctr_b200 import engine as E
    from deepctr_b200.layers import BilinearInteraction, SENETLayer
    E.clear_session()
    with pytest.raises(ValueError, match="at least 2 inputs"):
        SENETLayer().build([(None, 1, 4)])
    with pytest.raises(ValueError, match="at least 2 inputs"):
        BilinearInteraction().build([(None, 1, 4)])
    E.clear_session()
    se = SENETLayer(reduction_ratio=3, seed=5)
    se.build([(None, 1, 6)] * 2)
    assert [(w.name, w.shape) for w in se.weights] == [("senet_layer/W_1", (2, 1)), ("senet_layer/W_2", (1, 2))]
    assert se.compute_mask(None) == [None, None]
    assert se.compute_output_shape([(None, 1, 6)] * 2) == [(None, 1, 6)] * 2
    assert E.Lambda(lambda v: v).name == "lambda_1"          # the nested Lambda took `lambda`
    bi = BilinearInteraction(bilinear_type="interaction", seed=7)
    bi.build([(None, 1, 5)] * 4)
    assert [w.name for w in bi.weights] == ["bilinear_interaction/bilinear_weight%d_%d" % p
                                            for p in [(0, 1), (0, 2), (0, 3), (1, 2), (1, 3), (2, 3)]]
    assert bi.compute_output_shape([(None, 1, 5)] * 4) == (None, 6, 5)
    cfg = bi.get_config()
    assert (cfg["bilinear_type"], cfg["seed"]) == ("interaction", 7)
    cfg = SENETLayer(reduction_ratio=2, seed=9).get_config()
    assert (cfg["reduction_ratio"], cfg["seed"]) == (2, 9)


def _places(model):
    return sorted(((pl.n, pl.P, pl.E, pl.ndense, pl.ld, k) for pl, k in model.planner.dnn_places.values()),
                  key=lambda t: t[-1])


def test_dnn_input_placement_is_planned_for_fibinet_only():
    from deepctr_b200 import engine as E, inputs as I, models as M
    from deepctr_b200 import feature_column as FC
    cols = [FC.SparseFeat("C%d" % i, 30, 8) for i in range(6)] + [FC.DenseFeat("I%d" % i, 1) for i in range(3)]
    E.clear_session()
    # P = 15, 2 x 15 x 8 = 240 columns of pairs + 3 dense, padded to 244
    assert _places(M.FiBiNET(cols, cols)) == [(2, 15, 8, 3, 244, 0), (2, 15, 8, 3, 244, 1)]
    E.clear_session()
    assert _places(M.FiBiNET(cols[:6], cols[:6], dnn_hidden_units=())) == [(2, 15, 8, 0, 240, 0), (2, 15, 8, 0, 240, 1)]
    for builder in ("DeepFM", "NFM", "AFM"):
        E.clear_session()
        c = cols[:6] if builder == "AFM" else cols
        assert getattr(M, builder)(c, c).planner.dnn_places == {}, builder
    I.DNN_INPUT_PLACEMENT = False
    try:
        E.clear_session()
        assert M.FiBiNET(cols, cols).planner.dnn_places == {}
    finally:
        I.DNN_INPUT_PLACEMENT = True


def test_dnn_input_placement_needs_the_concat_pattern():
    """A bilinear output that also reaches another layer, or is not concatenated with its sibling, is not placed."""
    from deepctr_b200 import engine as E, models as M
    from deepctr_b200 import feature_column as FC
    from deepctr_b200.engine import Dense, Flatten, Model
    from deepctr_b200.layers import BilinearInteraction, DNN, PredictionLayer
    from deepctr_b200.layers.utils import combined_dnn_input, concat_func, add_func
    from deepctr_b200.feature_column import build_input_features, input_from_feature_columns
    cols = [FC.SparseFeat("C%d" % i, 30, 4) for i in range(4)]
    E.clear_session()
    feats = build_input_features(cols)
    embs, dense = input_from_feature_columns(feats, cols, 0, 1024)
    a = BilinearInteraction("all")(embs)
    b = BilinearInteraction("all")(embs)
    x = combined_dnn_input([Flatten()(concat_func([a, b]))], dense)
    side = Dense(1, use_bias=False)(Flatten()(a))                # a second consumer of `a`
    out = PredictionLayer()(add_func([Dense(1, use_bias=False)(DNN((8,))(x)), side]))
    assert Model(list(feats.values()), out).planner.dnn_places == {}
