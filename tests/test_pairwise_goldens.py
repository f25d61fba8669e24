"""CPU: NFM / AFM and their layers (BiInteractionPooling, AFMLayer) against fixtures the reference's own
layer and builder code produced (tests/golden/generate_pairwise.py):

1. the CPU restatement of tests/pairwise_oracle.py (built on oracle/) reproduces every layer output, model logit,
   prediction, loss and gradient;
2. the deepctr_b200 builders create the reference's weight set and graph (names, shapes, order, planner slots),
   and have the reference's keyword defaults;
3. the documented shape limits of the fused AFM kernels and AFM's DenseFeat refusal raise ValueError.
"""
import glob
import inspect
import json
import os

import numpy as np
import pytest
import torch

import golden_models as G
from test_reference_builders_dropin import signature, builder_args

HERE = os.path.dirname(os.path.abspath(__file__))
LAYERS = os.path.join(HERE, "golden", "pairwise")
MODELS = os.path.join(HERE, "golden", "models_pairwise")
BUILDERS_JSON = os.path.join(HERE, "golden", "reference_builders_pairwise.json")
LAYER_CASES = sorted(os.path.basename(p)[:-4] for p in glob.glob(os.path.join(LAYERS, "*.npz")))
MODEL_CASES = sorted(os.path.basename(p)[:-4] for p in glob.glob(os.path.join(MODELS, "*.npz")))


def load_layer(name):
    d = np.load(os.path.join(LAYERS, name + ".npz"))
    meta = json.loads(str(d["meta"]))
    return meta, {k: d[k] for k in d.files if k != "meta"}


class Fixture(G.Fixture):
    """golden_models.Fixture read from tests/golden/models_pairwise/."""

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


def oracle_weights(fx, requires_grad=False):
    """golden_models.oracle_weights plus the AFMLayer weights (one dict per layer, in graph order)."""
    W, leaves = G.oracle_weights(fx, requires_grad)

    def t(key):
        v = torch.tensor(fx.w[key], requires_grad=requires_grad and key in fx.g)
        leaves[key] = v
        return v
    W["afm"] = [{k: t("%s/%s" % (name, k)) for k in ("attention_W", "attention_b", "projection_h", "projection_p")}
                for name in fx.layer_names("AFMLayer")]
    return W, leaves


def oracle_forward(fx, W):
    import pairwise_oracle as PO
    from deepctr_b200 import feature_column as FC
    x = fx.inputs()
    lin, dnn = G.columns(fx, "linear", FC), G.columns(fx, "dnn", FC)
    if fx.builder == "NFM":
        return PO.nfm(x, lin, dnn, W, task=fx.task)
    kw = fx.kwargs
    fm_group = kw.get("fm_group", "default_group")
    return PO.afm_model(x, lin, dnn, W, fm_group=tuple(fm_group) if isinstance(fm_group, list) else fm_group,
                        use_attention=kw.get("use_attention", True), task=fx.task)


def build(fx):
    from deepctr_b200 import engine as E
    from deepctr_b200 import models as M
    args, kw = builder_args(fx)
    E.clear_session()
    return getattr(M, fx.builder)(*args, **kw)


def test_fixture_sets():
    assert len(LAYER_CASES) >= 6 and len(MODEL_CASES) >= 4
    assert set(Fixture(n).builder for n in MODEL_CASES) == {"NFM", "AFM"}


@pytest.mark.parametrize("name", LAYER_CASES)
def test_oracle_matches_reference_layer(name):
    import pairwise_oracle as PO
    meta, d = load_layer(name)
    x = torch.tensor(d["x"], requires_grad=True)
    if meta["layer"] == "AFMLayer":
        ws = {k: torch.tensor(d["w_" + k], requires_grad=True)
              for k in ("attention_W", "attention_b", "projection_h", "projection_p")}
        out = PO.afm(x, **ws)
    else:
        ws = {}
        out = PO.bi_interaction(x)
    np.testing.assert_allclose(out.detach().numpy(), d["out"], rtol=1e-5, atol=1e-6)
    (out * torch.as_tensor(d["dout"])).sum().backward()
    np.testing.assert_allclose(x.grad.numpy(), d["gx"], rtol=1e-4, atol=1e-6)
    for k, v in ws.items():
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
    for key, want in fx.g.items():
        if G._ignored(key):
            assert not np.any(want), key
            continue
        leaf = leaves[key]
        got = leaf.grad.numpy() if leaf.grad is not None else np.zeros_like(want)
        np.testing.assert_allclose(got, want, rtol=1e-4, atol=1e-4 * float(np.abs(want).max()) + 1e-7, err_msg=key)


@pytest.mark.parametrize("name", MODEL_CASES)
def test_builders_create_the_reference_weight_set(name):
    fx = Fixture(name)
    model = build(fx)
    wm = G.weight_map(fx, model)
    assert len(wm) == len([k for k in fx.w if not G._ignored(k)])
    for key, w in wm.items():
        assert w.trainable == (key in fx.g), key


@pytest.mark.parametrize("name", MODEL_CASES)
def test_builder_graph_is_the_reference_graph(name):
    with open(BUILDERS_JSON) as f:
        want = json.load(f)["signatures"][name]
    got = signature(build(Fixture(name)))
    assert want["inputs"] == got["inputs"]
    assert want["weights"] == got["weights"]           # in order: AFM looks up embeddings before the linear part
    assert want["slots"] == got["slots"] and want["fast"] == got["fast"]
    assert sorted(want["layers"]) == sorted(got["layers"])


def test_reference_default_arguments_are_the_same():
    from deepctr_b200 import models as M
    with open(BUILDERS_JSON) as f:
        ref = json.load(f)["defaults"]
    assert sorted(ref) == ["AFM", "NFM"]
    for name, params in ref.items():
        mine = inspect.signature(getattr(M, name))
        assert [k for k, _ in params] == list(mine.parameters), name
        for k, d in params:
            assert d == repr(mine.parameters[k].default), (name, k)


def test_afm_rejects_dense_features():
    from deepctr_b200 import engine as E
    from deepctr_b200 import feature_column as FC
    from deepctr_b200 import models as M
    cols = [FC.SparseFeat("a", 10, 4), FC.SparseFeat("b", 10, 4), FC.DenseFeat("d", 1)]
    E.clear_session()
    with pytest.raises(ValueError, match="DenseFeat is not supported"):
        M.AFM(cols, cols)


@pytest.mark.parametrize("nfields,dim,factor", [(65, 4, 4), (3, 33, 4), (3, 8, 17), (3, 8, 0)])
def test_afm_unsupported_shapes_raise(nfields, dim, factor):
    from deepctr_b200 import engine as E
    from deepctr_b200.layers import AFMLayer
    E.clear_session()
    with pytest.raises(ValueError):
        AFMLayer(attention_factor=factor).build([(None, 1, dim)] * nfields)


def test_afm_layer_reference_checks():
    from deepctr_b200.layers import AFMLayer
    with pytest.raises(ValueError, match="at least 2 inputs"):
        AFMLayer().build([(None, 1, 4)])
    with pytest.raises(ValueError, match="same shapes"):
        AFMLayer().build([(None, 1, 4), (None, 1, 8)])
    with pytest.raises(ValueError, match="embedding_size"):
        AFMLayer().build([(None, 2, 4), (None, 2, 4)])
    with pytest.raises(ValueError, match="list of inputs"):
        AFMLayer().compute_output_shape((None, 1, 4))
    cfg = AFMLayer(attention_factor=3, l2_reg_w=0.5, dropout_rate=0.1, seed=7).get_config()
    assert {k: cfg[k] for k in ("attention_factor", "l2_reg_w", "dropout_rate", "seed")} == \
        {"attention_factor": 3, "l2_reg_w": 0.5, "dropout_rate": 0.1, "seed": 7}


def test_afm_layer_weights_and_nested_names():
    """attention_W / attention_b / projection_h / projection_p with the reference's shapes and regularizer, and the
    nested Dropout / Lambda take the next `dropout` / `lambda` names as in Keras."""
    from deepctr_b200 import engine as E
    from deepctr_b200.layers import AFMLayer, BiInteractionPooling
    from deepctr_b200.layers.normalization import Dropout
    E.clear_session()
    layer = AFMLayer(attention_factor=5, l2_reg_w=0.25)
    layer.build([(None, 1, 6)] * 3)
    assert [(w.name, w.shape) for w in layer.weights] == [
        ("afm_layer/attention_W", (6, 5)), ("afm_layer/attention_b", (5,)), ("afm_layer/projection_h", (5, 1)),
        ("afm_layer/projection_p", (6, 1))]
    assert layer.attention_W.l2 == 0.25 and layer.projection_p.l2 == 0.0
    assert Dropout(0.1).name == "dropout_1" and E.Lambda(lambda v: v).name == "lambda_1"
    bi = BiInteractionPooling()
    assert bi.compute_output_shape((None, 7, 6)) == (None, 1, 6)
    with pytest.raises(ValueError, match="expect to be 3 dimensions"):
        bi.build((None, 6))
