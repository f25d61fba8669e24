"""CPU: FiBiNET and its layers (SENETLayer, BilinearInteraction) against fixtures the reference's own layer and
builder code produced (tests/golden/generate_fibinet.py):

1. the CPU restatement of tests/fibinet_oracle.py (built on oracle/) reproduces every layer output and, with the
   checks shared by every family (model_golden_checks), every model fixture, weight set, graph and keyword default;
2. the documented shape limits of the SENET / bilinear kernels raise ValueError, an unknown bilinear_type raises
   NotImplementedError;
3. the DNN-input placement is planned for FiBiNET's graph, and only there.
"""

import pytest

import golden_models as G
import model_golden_checks as C

T = C.model_tests("fibinet")
test_oracle_matches_reference_model = T.oracle
test_builder_creates_the_reference_weight_set = T.weight_set
test_builder_graph_is_the_reference_graph = T.graph
test_reference_default_arguments_are_the_same = T.defaults
L = C.layer_tests("fibinet")
test_oracle_matches_reference_layer = L.oracle


def test_fixture_sets():
    C.check_fixture_set(G.FAMILIES["fibinet"])
    L.fixture_set()
    fam = G.FAMILIES["fibinet"]
    assert {fam.fixture(n).kwargs["bilinear_type"] for n in fam.cases} == {"all", "each", "interaction"}


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
