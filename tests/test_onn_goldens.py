"""CPU: ONN against fixtures the reference's own builder and feature-column code produced
(tests/golden/generate_onn.py): the model fixtures, weight sets, graphs and keyword defaults with the checks shared
by every family (model_golden_checks); the reference's build-time errors, the tables the model holds, the planner's
claim on the field-aware lookups, K.sum's shape inference and the update policies ONN rejects.
"""
import pytest

import model_golden_checks as C
import onn_family  # noqa: F401  (registers the "onn" fixture family)

T = C.model_tests("onn")
test_oracle_matches_reference_model = T.oracle
test_builder_creates_the_reference_weight_set = T.weight_set
test_builder_graph_is_the_reference_graph = T.graph
test_reference_default_arguments_are_the_same = T.defaults
test_fixture_set = T.fixture_set


def _columns(n_sparse=4, n_dense=2, dim=4, varlen=False):
    from deepctr_b200 import feature_column as FC
    cols = [FC.SparseFeat("C%d" % i, 30, dim) for i in range(n_sparse)] + [FC.DenseFeat("I%d" % i, 1)
                                                                             for i in range(n_dense)]
    if varlen:
        cols.append(FC.VarLenSparseFeat(FC.SparseFeat("S", 12, dim), maxlen=3, combiner="mean"))
    return cols


def _onn(cols, **kw):
    from deepctr_b200 import engine as E, models as M
    E.clear_session()
    return M.ONN(cols, cols, **kw)


def test_mismatched_embedding_dims_are_a_build_time_error():
    from deepctr_b200 import feature_column as FC
    cols = [FC.SparseFeat("a", 10, 4), FC.SparseFeat("b", 10, 8)]
    with pytest.raises(ValueError, match="embedding dimensions 4 and 8"):
        _onn(cols)


def test_embedding_name_other_than_name_raises_key_error_like_the_reference():
    """onn.py's feature_embedding indexes the table dict (keyed by embedding_name) by fc.name."""
    from deepctr_b200 import feature_column as FC
    cols = [FC.SparseFeat("a", 10, 4, embedding_name="shared_a"), FC.SparseFeat("b", 10, 4)]
    with pytest.raises(KeyError):
        _onn(cols)


@pytest.mark.parametrize("n_sparse,dim", [(1, 4), (65, 4), (3, 65)])
def test_field_and_dimension_limits(n_sparse, dim):
    with pytest.raises(ValueError):
        _onn(_columns(n_sparse=n_sparse, dim=dim))


@pytest.mark.parametrize("varlen", [False, True])
def test_only_off_diagonal_tables_are_weights(varlen):
    cols = _columns(varlen=varlen)
    model = _onn(cols)
    names = [f.name for f in cols if hasattr(f, "embedding_name")]
    tabs = [w.name for w in model.weights if w.name.startswith("sparse_emb_")]
    want = []
    for i in range(len(names)):
        for j in range(i + 1, len(names)):
            want += ["sparse_emb_%s_%s/embeddings" % (names[i], names[j]),
                     "sparse_emb_%s_%s/embeddings" % (names[j], names[i])]
    assert tabs == want                     # pair by pair, (i -> j) then (j -> i); no sparse_emb_<a>_<a>


@pytest.mark.parametrize("reduce_sum", [False, True])
@pytest.mark.parametrize("varlen", [False, True])
def test_planner_claims_the_field_aware_lookups(reduce_sum, varlen):
    from deepctr_b200 import engine as E
    model = _onn(_columns(varlen=varlen), reduce_sum=reduce_sum)
    plan = model.planner.ffm
    F = 5 if varlen else 4
    assert plan is not None and plan.F == F and plan.P == F * (F - 1) // 2 and plan.reduce_sum == reduce_sum
    assert plan.width == plan.P * (1 if reduce_sum else 4)
    # the main gather keeps only the linear term's dim-1 lookups
    assert all(s.emb.name.startswith("linear0sparse_") for s in model.planner.slots)
    assert not model.planner.main
    served = E.Lambda if reduce_sum else E.Multiply
    assert all(isinstance(n.layer, served) for n in plan.pair_nodes)


def test_k_sum_lambda_shape_and_marker():
    from deepctr_b200 import backend as K, engine as E
    E.clear_session()
    x = E.Input(shape=(1, 4), name="x")
    lam = E.Lambda(lambda t: K.sum(t, axis=-1))
    y = lam(x)
    assert y.shape == (None, 1) and lam.reduces_last_axis
    lam2 = E.Lambda(lambda t: K.sum(t, axis=1, keepdims=True))
    assert lam2(x).shape == (None, 1, 4) and not lam2.reduces_last_axis
    lam3 = E.Lambda(lambda t: t)
    assert lam3(x).shape == (None, 1, 4) and not lam3.reduces_last_axis


@pytest.mark.parametrize("mode,opt", [("sparse_deterministic", "sgd"), ("sparse", "adagrad")])
def test_sorted_and_rowwise_adagrad_updates_are_rejected(mode, opt):
    from deepctr_b200 import engine as E
    model = _onn(_columns(), l2_reg_embedding=0, l2_reg_linear=0)
    with pytest.raises(ValueError, match="field-aware tables"):
        model.compile(E.SGD(0.1) if opt == "sgd" else E.Adagrad(0.1), "binary_crossentropy", embedding_update=mode)


@pytest.mark.parametrize("mode", ["dense", "sparse"])
def test_dense_and_sparse_sgd_updates_are_accepted(mode):
    from deepctr_b200 import engine as E
    model = _onn(_columns(), l2_reg_embedding=0, l2_reg_linear=0)
    model.compile(E.SGD(0.1), "binary_crossentropy", embedding_update=mode)
    plan = model.planner.ffm
    assert all(t.embeddings.sparse_grad == (mode == "sparse") for _, t in plan.tables)


def test_other_builders_plan_no_field_aware_products():
    from deepctr_b200 import engine as E, models as M
    cols = _columns()
    for b in ("DeepFM", "NFM", "FwFM"):
        E.clear_session()
        assert getattr(M, b)(cols, cols).planner.ffm is None, b
