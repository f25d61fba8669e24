"""CPU: IFM and DIFM against fixtures the reference's own builder and feature-column code produced
(tests/golden/generate_ifm.py): the model fixtures, weight sets, graphs and keyword defaults with the checks
shared by every family (model_golden_checks); the shape of the varlen fixtures, the reference's checks and
messages, the field-count check of the refined linear term, the Lambda shape inference of the two refine lambdas,
and what ops.softmax still rejects.
"""
import pytest
import torch

import golden_models as G
import model_golden_checks as C

T = C.model_tests("ifm")
test_oracle_matches_reference_model = T.oracle
test_builder_creates_the_reference_weight_set = T.weight_set
test_builder_graph_is_the_reference_graph = T.graph
test_reference_default_arguments_are_the_same = T.defaults


def _columns(n_sparse=4, n_dense=2, dim=4):
    from deepctr_b200 import feature_column as FC
    return ([FC.SparseFeat("C%d" % i, 30, dim) for i in range(n_sparse)] +
            [FC.DenseFeat("I%d" % i, 1) for i in range(n_dense)])


def test_fixture_sets():
    C.check_fixture_set(G.FAMILIES["ifm"])
    # the varlen fixtures count their pooled sequences as fields: F = 3 sparse + 4 varlen
    for name in ("ifm_varlen", "difm_two_heads_varlen"):
        fx = G.FAMILIES["ifm"].fixture(name)
        assert fx.w["dense/kernel" if fx.builder == "IFM" else "dense_1/kernel"].shape[1] == 7, name


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
    model = G.build(G.FAMILIES["ifm"].fixture("ifm_criteo"))
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
