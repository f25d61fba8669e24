"""CPU: FwFM / DeepFEFM and their layers (FwFMLayer, FEFMLayer) against fixtures the reference's own layer and builder
code produced (tests/golden/generate_fefm.py):

1. the CPU restatement of tests/fefm_oracle.py (built on oracle/) reproduces every layer output, model logit,
   prediction, loss and gradient;
2. the deepctr_b200 builders create the reference's weight set and graph (names, shapes, order, planner slots) -
   only what is reachable from the output - and have the reference's keyword defaults;
3. the reference's build-time checks and messages, the documented kernel limits (ValueError) and DeepFEFM's
   NotImplementedError branch;
4. the placement of DeepFEFM's FEFM scores in the DNN input is planned for DeepFEFM's graph, and only there.
"""
import glob
import inspect
import itertools
import json
import os

import numpy as np
import pytest
import torch

import golden_models as G
from test_reference_builders_dropin import signature, builder_args

HERE = os.path.dirname(os.path.abspath(__file__))
LAYERS = os.path.join(HERE, "golden", "fefm")
MODELS = os.path.join(HERE, "golden", "models_fefm")
BUILDERS_JSON = os.path.join(HERE, "golden", "reference_builders_fefm.json")
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
    """golden_models.Fixture read from tests/golden/models_fefm/."""

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
    """golden_models.oracle_weights plus W['fwfm'] (each FwFMLayer's strengths, in creation order) or W['fefm']
    (the FEFMLayer's P matrices, in itertools.combinations order)."""
    W, leaves = G.oracle_weights(fx, requires_grad)

    def t(key):
        v = torch.tensor(fx.w[key], requires_grad=requires_grad and key in fx.g)
        leaves[key] = v
        return v
    W["fwfm"] = [t(n + "/field_pair_strengths") for n in fx.layer_names("FwFMLayer")]
    for n in fx.layer_names("FEFMLayer"):
        F = int(round((1 + np.sqrt(1 + 8 * len([k for k in fx.w if k.startswith(n + "/")]))) / 2))
        W["fefm"] = [t("%s/field_embeddings%d-%d" % (n, i, j)) for i, j in itertools.combinations(range(F), 2)]
    return W, leaves


def oracle_forward(fx, W):
    import fefm_oracle as FO
    from deepctr_b200 import feature_column as FC
    lin, dnn = G.columns(fx, "linear", FC), G.columns(fx, "dnn", FC)
    kw = fx.kwargs
    if fx.builder == "FwFM":
        return FO.fwfm_model(fx.inputs(), lin, dnn, W, fm_group=tuple(kw.get("fm_group", ("default_group",))),
                             task=fx.task)
    return FO.deepfefm(fx.inputs(), lin, dnn, W, use_fefm=kw.get("use_fefm", True),
                       use_linear=kw.get("use_linear", True),
                       use_fefm_embed_in_dnn=kw.get("use_fefm_embed_in_dnn", True),
                       exclude_feature_embed_in_dnn=kw.get("exclude_feature_embed_in_dnn", False), task=fx.task)


def build(fx):
    from deepctr_b200 import engine as E
    from deepctr_b200 import models as M
    args, kw = builder_args(fx)
    E.clear_session()
    return getattr(M, fx.builder)(*args, **kw)


def test_fixture_sets():
    assert len(LAYER_CASES) == 6 and len(MODEL_CASES) == 10
    assert {Fixture(n).builder for n in MODEL_CASES} == {"FwFM", "DeepFEFM"}
    assert {Fixture(n).task for n in MODEL_CASES} == {"binary", "regression"}


@pytest.mark.parametrize("name", LAYER_CASES)
def test_oracle_matches_reference_layer(name):
    import fefm_oracle as FO
    meta, d = load_layer(name)
    x = torch.tensor(d["x"], requires_grad=True)
    ws = [torch.tensor(d["w_" + k], requires_grad=True) for k in layer_weight_names(d)]
    out = FO.fwfm(x, ws[0]) if meta["layer"] == "FwFMLayer" else FO.fefm(x, ws)
    np.testing.assert_allclose(out.detach().numpy(), d["out"], rtol=1e-5, atol=1e-6)
    (out * torch.as_tensor(d["dout"])).sum().backward()
    np.testing.assert_allclose(x.grad.numpy(), d["gx"], rtol=1e-4, atol=1e-6)
    for k, v in zip(layer_weight_names(d), ws):
        np.testing.assert_allclose(v.grad.numpy(), d["g_" + k], rtol=1e-4, atol=1e-6, err_msg=k)
    if meta["layer"] == "FwFMLayer":
        g = d["g_field_pair_strengths"]
        assert not np.any(np.tril(g)), "the strengths' gradient is 0 on and below the diagonal"


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
    # the fixture lists weights in creation order, a model in graph order: the two differ where a group's
    # FwFMLayer is built before the next group's embeddings (fwfm_two_groups).  The graph order itself is
    # pinned against the reference builder's in test_builder_graph_is_the_reference_graph.
    mine = [w.name for w in model.weights if not G._ignored(w.name)]
    ref = [k for k in fx.w if not G._ignored(k)]
    assert sorted(mine) == sorted(ref)
    if fx.name != "fwfm_two_groups":
        assert mine == ref, "weight order"
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


def test_unreachable_branches_hold_no_weights():
    """With dnn_hidden_units=() the reference still creates a DNN and a Dense(1) (and, without use_linear, the
    linear part); they are off the output path, so neither graph holds them."""
    fx = Fixture("deepfefm_linear_fefm")
    model = build(fx)
    assert not any(type(l).__name__ in ("DNN", "Dense") for l in model.layers)
    assert not any("dense" in w.name or w.name.startswith("dnn") for w in model.weights)
    model = build(Fixture("deepfefm_no_linear"))
    assert not any(w.name.startswith("linear") for w in model.weights)


def test_reference_default_arguments_are_the_same():
    from deepctr_b200 import models as M
    with open(BUILDERS_JSON) as f:
        ref = json.load(f)["defaults"]
    assert sorted(ref) == ["DeepFEFM", "FwFM"]
    for b in ref:
        mine = inspect.signature(getattr(M, b))
        assert [k for k, _ in ref[b]] == list(mine.parameters), b
        for k, d in ref[b]:
            assert d == repr(mine.parameters[k].default), (b, k)


def test_deepfefm_unsupported_branch_raises():
    from deepctr_b200 import engine as E, models as M
    from deepctr_b200 import feature_column as FC
    cols = [FC.SparseFeat("C%d" % i, 30, 4) for i in range(4)]
    E.clear_session()
    with pytest.raises(NotImplementedError):
        M.DeepFEFM(cols, cols, dnn_hidden_units=(), use_fefm=False, use_linear=False)


@pytest.mark.parametrize("nfields,dim", [(65, 4), (3, 65), (1, 4)])
def test_unsupported_shapes_raise(nfields, dim):
    from deepctr_b200 import engine as E
    from deepctr_b200.layers import FEFMLayer, FwFMLayer
    E.clear_session()
    with pytest.raises(ValueError, match="FwFMLayer supports 2 to 64 fields and embedding_size 1 to 64"):
        FwFMLayer(num_fields=nfields).build((None, nfields, dim))
    with pytest.raises(ValueError, match="FEFMLayer supports 2 to 64 fields and embedding_size 1 to 64"):
        FEFMLayer(1e-5).build((None, nfields, dim))


def test_layer_reference_checks_weights_and_config():
    from deepctr_b200 import engine as E
    from deepctr_b200.layers import FEFMLayer, FwFMLayer
    E.clear_session()
    with pytest.raises(ValueError) as e:
        FwFMLayer(num_fields=3).build((None, 12))
    assert str(e.value) == "Unexpected inputs dimensions  2," + " " * 29 + "expect to be 3 dimensions"
    with pytest.raises(ValueError) as e:
        FwFMLayer(num_fields=3).build((None, 4, 8))
    assert str(e.value) == "Mismatch in number of fields 3 and" + " " * 18 + "concatenated embeddings dims 4"
    with pytest.raises(ValueError) as e:
        FEFMLayer(1e-5).build((None, 4, 8, 1))
    assert str(e.value) == "Unexpected inputs dimensions  4," + " " * 32 + "expect to be 3 dimensions"
    E.clear_session()
    fw = FwFMLayer(num_fields=3, regularizer=1e-4)
    fw.build((None, 3, 8))
    assert [(w.name, w.shape) for w in fw.weights] == [("fw_fm_layer/field_pair_strengths", (3, 3))]
    assert fw.weights[0].regularizer.l2 == pytest.approx(1e-4)
    assert fw.compute_output_shape((None, 3, 8)) == (None, 1)
    cfg = fw.get_config()
    assert (cfg["num_fields"], cfg["regularizer"]) == (3, 1e-4)
    fe = FEFMLayer(regularizer=2e-5)
    fe.build((None, 4, 5))
    assert [(w.name, w.shape) for w in fe.weights] == [("fefm_layer/field_embeddings%d-%d" % p, (5, 5))
                                                       for p in itertools.combinations(range(4), 2)]
    assert fe.compute_output_shape((None, 4, 5)) == (None, 6)
    assert fe.get_config()["regularizer"] == 2e-5


def test_fefm_placement_is_planned_for_deepfefm_only():
    """DeepFEFM's FEFM scores get P columns behind the dense tail of the gather buffer only where its DNN input is
    concat([combined_dnn_input, scores]); every other model and ablation keeps its row pitch."""
    from deepctr_b200 import engine as E, inputs as I, models as M
    from deepctr_b200 import feature_column as FC
    cols = [FC.SparseFeat("C%d" % i, 30, 8) for i in range(6)] + [FC.DenseFeat("I%d" % i, 1) for i in range(3)]

    def plan(model):
        p = model.planner
        return p.main_width, p.main_ld, sorted(p.fefm_places.values())
    E.clear_session()
    # 6 x 8 = 48 embedding columns + 3 dense + P = 15 scores = 66, padded to 68
    assert plan(M.DeepFEFM(cols, cols)) == (48, 68, [15])
    E.clear_session()
    assert plan(M.DeepFEFM(cols[:6], cols[:6])) == (48, 64, [15])           # no dense features: 48 + 15 -> 64
    for kw in (dict(exclude_feature_embed_in_dnn=True), dict(use_fefm_embed_in_dnn=False),
               dict(dnn_hidden_units=())):
        E.clear_session()
        assert plan(M.DeepFEFM(cols, cols, **kw)) == (48, 52, []), kw
    for builder in ("DeepFM", "NFM", "FiBiNET", "FwFM"):
        E.clear_session()
        model = getattr(M, builder)(cols, cols)
        assert model.planner.fefm_places == {}, builder
        assert model.planner.main_ld == 52, builder          # 48 + 3 dense, padded to 4
    I.DNN_INPUT_PLACEMENT = False
    try:
        E.clear_session()
        assert plan(M.DeepFEFM(cols, cols)) == (48, 52, [])
    finally:
        I.DNN_INPUT_PLACEMENT = True
