"""CPU: IFM and DIFM against fixtures the reference's own builder and feature-column code produced
(tests/golden/generate_ifm.py):

1. the CPU restatement of tests/ifm_oracle.py (built on oracle/) reproduces every model logit, prediction, loss and
   gradient;
2. the deepctr_b200 builders create the reference's weight set and graph (names, shapes, order, planner slots) and
   have the reference's keyword defaults;
3. the reference's checks and messages, the field-count check of the refined linear term, the Lambda shape inference
   of the two refine lambdas, and what ops.softmax still rejects.
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
MODELS = os.path.join(HERE, "golden", "models_ifm")
BUILDERS_JSON = os.path.join(HERE, "golden", "reference_builders_ifm.json")
MODEL_CASES = sorted(os.path.basename(p)[:-4] for p in glob.glob(os.path.join(MODELS, "*.npz")))


class Fixture(G.Fixture):
    """golden_models.Fixture read from tests/golden/models_ifm/."""

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
    """golden_models.oracle_weights plus W['m_kernels'], the Dense(F) kernels in creation order."""
    W, leaves = G.oracle_weights(fx, requires_grad)
    W["m_kernels"] = []
    for n in fx.layer_names("Dense"):
        W["m_kernels"].append(leaves[n + "/kernel"] if n + "/kernel" in leaves else
                              torch.tensor(fx.w[n + "/kernel"], requires_grad=requires_grad))
        leaves[n + "/kernel"] = W["m_kernels"][-1]
    return W, leaves


def oracle_forward(fx, W):
    import ifm_oracle as IO
    from deepctr_b200 import feature_column as FC
    kw = fx.kwargs
    args = (fx.inputs(), G.columns(fx, "linear", FC), G.columns(fx, "dnn", FC), W)
    if fx.builder == "IFM":
        return IO.ifm(*args, task=fx.task)
    return IO.difm(*args, att_embedding_size=kw.get("att_embedding_size", 8), att_head_num=kw.get("att_head_num", 8),
                   att_res=kw.get("att_res", True), task=fx.task)


def build(fx):
    from deepctr_b200 import engine as E
    from deepctr_b200 import models as M
    args, kw = builder_args(fx)
    E.clear_session()
    return getattr(M, fx.builder)(*args, **kw)


def _columns(n_sparse=4, n_dense=2, dim=4):
    from deepctr_b200 import feature_column as FC
    return ([FC.SparseFeat("C%d" % i, 30, dim) for i in range(n_sparse)] +
            [FC.DenseFeat("I%d" % i, 1) for i in range(n_dense)])


def test_fixture_sets():
    assert len(MODEL_CASES) == 6
    assert {Fixture(n).builder for n in MODEL_CASES} == {"IFM", "DIFM"}
    assert {Fixture(n).task for n in MODEL_CASES} == {"binary", "regression"}
    # the varlen fixtures count their pooled sequences as fields: F = 3 sparse + 4 varlen
    for name in ("ifm_varlen", "difm_two_heads_varlen"):
        fx = Fixture(name)
        assert fx.w["dense/kernel" if fx.builder == "IFM" else "dense_1/kernel"].shape[1] == 7, name


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
    # (the fixture lists weights in creation order; the model's order, the graph's, is checked against the
    # reference-built graph in test_builder_graph_is_the_reference_graph)
    assert sorted(w.name for w in model.weights) == sorted(fx.w)
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
    assert sorted(ref) == ["DIFM", "IFM"]
    for b in ("IFM", "DIFM"):
        mine = inspect.signature(getattr(M, b))
        assert [k for k, _ in ref[b]] == list(mine.parameters), b
        for k, d in ref[b]:
            assert d == repr(mine.parameters[k].default), (b, k)


@pytest.mark.parametrize("builder", ["IFM", "DIFM"])
def test_reference_errors(builder):
    from deepctr_b200 import engine as E, models as M
    cols = _columns()
    E.clear_session()
    with pytest.raises(ValueError) as e:
        getattr(M, builder)(cols, cols, dnn_hidden_units=())
    assert str(e.value) == "dnn_hidden_units is null!"
    dense_only = _columns(n_sparse=0)
    E.clear_session()
    with pytest.raises(ValueError) as e:
        getattr(M, builder)(dense_only, dense_only)
    assert str(e.value) == "there are no sparse features"


@pytest.mark.parametrize("builder", ["IFM", "DIFM"])
def test_linear_and_fm_field_counts_must_match(builder):
    """The reference broadcasts m over the linear lookups when one count is 1 and fails inside TensorFlow otherwise:
    here a different count of linear sparse features is a ValueError at build time that names both counts."""
    from deepctr_b200 import engine as E, models as M
    cols = _columns(n_sparse=4)
    E.clear_session()
    with pytest.raises(ValueError, match="has 4 field weights but the linear part has 3 sparse features"):
        getattr(M, builder)(cols[:3] + cols[4:], cols)
    E.clear_session()
    getattr(M, builder)(cols[4:], cols)           # no linear sparse features: nothing is refined


def test_difm_interacting_limit():
    """DIFM inherits InteractingLayer's limit F * att_embedding_size * att_head_num <= 3072: F <= 48 at the defaults."""
    from deepctr_b200 import engine as E, models as M
    E.clear_session()
    M.DIFM([], _columns(n_sparse=48, n_dense=0), dnn_hidden_units=(8,))
    E.clear_session()
    with pytest.raises(ValueError, match="InteractingLayer supports"):
        M.DIFM([], _columns(n_sparse=49, n_dense=0), dnn_hidden_units=(8,))


def test_refine_lambdas_have_one_output_of_the_broadcast_shape():
    """A Lambda over [x, m] without output_shape has the shape of its highest-rank input: IFM's refined FM input is
    one [B, F, E] tensor, and the softmax Lambda keeps [B, F]."""
    from deepctr_b200 import engine as E, ops
    E.clear_session()
    x, m = E.Input((5, 4), name="x"), E.Input((5,), name="m")
    refined = E.Lambda(lambda v: ops.scale_fields(v[0], v[1]))([x, m])
    assert isinstance(refined, E.KTensor) and refined.shape == (None, 5, 4)
    assert E.Lambda(lambda v: ops.softmax(v, dim=1, scale=5))(m).shape == (None, 5)
    assert E.Lambda(lambda v: v, output_shape=(None, 3))([x, m]).shape == (None, 3)
    model = build(Fixture("ifm_criteo"))
    lambdas = [l for l in model.layers if isinstance(l, E.Lambda)]
    assert len(lambdas) == 2
    from deepctr_b200.layers.utils import RefineWeight
    refine = [l for l in model.layers if isinstance(l, RefineWeight)]
    assert len(refine) == 1 and refine[0].compute_output_shape([(None, 1, 6), (None, 6)]) == (None, 1, 6)


def test_softmax_other_ranks_and_axes_still_raise():
    from deepctr_b200 import engine as E, ops
    with pytest.raises(NotImplementedError):
        ops.softmax(E.Var(torch.zeros(2, 3, 4)))
    with pytest.raises(NotImplementedError):
        ops.softmax(E.Var(torch.zeros(2, 3)), dim=0)
    with pytest.raises(NotImplementedError):
        ops.softmax(E.Var(torch.zeros(6)))


def test_linear_rows_are_not_fused_into_the_gather_when_refined():
    """The gather-epilogue row-sum of the linear lookups (lin_hint) is only for Linear reading the raw window: an IFM
    graph marks its linear lookups refined, and the row-wise paths that would fuse them refuse it."""
    from deepctr_b200 import engine as E, models as M
    cols = _columns(n_sparse=4, n_dense=0)
    E.clear_session()
    ifm = M.IFM(cols, cols, dnn_hidden_units=(8,))
    assert ifm.planner.lin_refined and not ifm.planner.lin_hint
    E.clear_session()
    assert not M.DeepFM(cols, cols).planner.lin_refined

    class _Opt(object):
        name = "adagrad"
    with pytest.raises(ValueError, match="sparse_feat_refine_weight"):
        ifm.planner.configure(_Opt(), "sparse_deterministic")
