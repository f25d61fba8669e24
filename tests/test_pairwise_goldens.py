"""CPU: NFM / AFM and their layers (BiInteractionPooling, AFMLayer) against fixtures the reference's own
layer and builder code produced (tests/golden/generate_pairwise.py):

1. the CPU restatement of tests/pairwise_oracle.py (built on oracle/) reproduces every layer output and, with the
   checks shared by every family (model_golden_checks), every model fixture;
2. the documented shape limits of the fused AFM kernels and AFM's DenseFeat refusal raise ValueError.
"""

import pytest

import golden_models as G
import model_golden_checks as C

T = C.model_tests("pairwise")
test_oracle_matches_reference_model = T.oracle
test_builders_create_the_reference_weight_set = T.weight_set
test_builder_graph_is_the_reference_graph = T.graph
test_reference_default_arguments_are_the_same = T.defaults
L = C.layer_tests("pairwise")
test_oracle_matches_reference_layer = L.oracle


def test_fixture_sets():
    C.check_fixture_set(G.FAMILIES["pairwise"])
    L.fixture_set()


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
