"""CPU: EDCN against fixtures the reference's own builder, layer and feature-column code produced
(tests/golden/generate_edcn.py): the model fixtures, weight sets, graphs and keyword defaults with the checks shared
by every family (model_golden_checks); the reference's build-time errors and prints, RegulationModule's and
BridgeModule's weights and get_config, Activation('softmax') shape inference, the planner's fused launches and the
descriptor layout of b2ctr_regulate.
"""
import ctypes

import numpy as np
import pytest

import model_golden_checks as C
import edcn_family  # noqa: F401  (registers the "edcn" fixture family)

T = C.model_tests("edcn")
test_oracle_matches_reference_model = T.oracle
test_builder_creates_the_reference_weight_set = T.weight_set
test_builder_graph_is_the_reference_graph = T.graph
test_reference_default_arguments_are_the_same = T.defaults
test_fixture_set = T.fixture_set

BRIDGES = ("pointwise_addition", "hadamard_product", "concatenation", "attention_pooling")


def _columns(n_sparse=4, dim=4, dense=False):
    from deepctr_b200 import feature_column as FC
    cols = [FC.SparseFeat("C%d" % i, 30, dim) for i in range(n_sparse)]
    return cols + ([FC.DenseFeat("I0", 1)] if dense else [])


def _edcn(cols, linear=None, **kw):
    from deepctr_b200 import engine as E, models as M
    E.clear_session()
    return M.EDCN(cols if linear is None else linear, cols, **kw)


@pytest.mark.parametrize("cross_num", [0, -1])
def test_cross_num_below_one_raises_the_reference_error(cross_num):
    with pytest.raises(ValueError, match="Cross layer num must > 0"):
        _edcn(_columns(), cross_num=cross_num)


def test_linear_column_missing_from_dnn_columns_raises_key_error():
    from deepctr_b200 import feature_column as FC
    with pytest.raises(KeyError):
        _edcn(_columns(), linear=_columns() + [FC.SparseFeat("extra", 10, 4)])


def test_dense_features_are_rejected():
    with pytest.raises(ValueError, match="DenseFeat is not supported"):
        _edcn(_columns(dense=True))


def test_mismatched_embedding_dims_are_a_build_time_error():
    from deepctr_b200 import feature_column as FC
    cols = [FC.SparseFeat("a", 10, 4), FC.SparseFeat("b", 10, 8)]
    with pytest.raises(ValueError, match="embedding dimensions 4 and 8"):
        _edcn(cols)


def test_unknown_bridge_type_names_it_and_the_valid_types():
    with pytest.raises(ValueError, match="'sum'.*pointwise_addition, hadamard_product, concatenation, "
                                         "attention_pooling"):
        _edcn(_columns(), bridge_type="sum")


def test_tau_zero_raises_the_reference_error():
    from deepctr_b200.layers import RegulationModule
    with pytest.raises(ValueError, match="RegulationModule tau can not be zero."):
        RegulationModule(0)
    with pytest.raises(ValueError, match="RegulationModule tau can not be zero."):
        _edcn(_columns(), tau=0)


def test_builder_prints_the_reference_lines(capsys):
    _edcn(_columns(), cross_num=2, bridge_type="hadamard_product")
    out = capsys.readouterr().out.splitlines()
    assert out[0] == "EDCN brige type:  hadamard_product"
    assert sum(line.startswith("CrossNet parameterization:") for line in out) == 2
    pairs = [line for line in out if line.startswith("KTensor") or "KTensor" in line]
    assert len(pairs) == 2                                 # print(cross_out, deep_out) per layer


def test_regulation_module_weight_config_and_shape():
    from deepctr_b200 import engine as E
    from deepctr_b200.layers import RegulationModule, custom_objects
    E.clear_session()
    x = E.Input(shape=(5, 4), name="x")
    reg = RegulationModule(tau=0.5)
    y = reg(x)
    assert y.shape == (None, 20)
    (w,) = reg.weights
    assert w.name == "%s/%s_field_weight" % (reg.name, reg.name) and tuple(w.shape) == (1, 5, 1)
    np.testing.assert_array_equal(w.value(), np.ones((1, 5, 1), np.float32))
    cfg = reg.get_config()
    assert cfg["tau"] == 2.0 and cfg["name"] == reg.name          # the reference stores and returns 1 / tau
    assert custom_objects["RegulationModule"] is RegulationModule


@pytest.mark.parametrize("bridge_type", BRIDGES)
def test_bridge_module_weights_and_config(bridge_type):
    from deepctr_b200 import engine as E
    from deepctr_b200.layers import BridgeModule, custom_objects
    E.clear_session()
    x, h = E.Input(shape=(12,), name="x"), E.Input(shape=(12,), name="h")
    br = BridgeModule(bridge_type, activation="relu")
    assert br([x, h]).shape == (None, 12)
    got = [(w.name, tuple(w.shape)) for w in br.weights]
    n = br.name
    want = {"concatenation": [(n + "/dense/kernel", (24, 12)), (n + "/dense/bias", (12,))],
            "attention_pooling": [("%s/%s/%s%d" % (n, s, k, i), (12, 12) if k == "kernel" else (12,))
                                  for s in ("dense_x", "dense_h") for k in ("kernel", "bias") for i in range(2)]}
    assert got == want.get(bridge_type, [])
    cfg = br.get_config()
    assert cfg["bridge_type"] == bridge_type and cfg["activation"] == "relu" and cfg["name"] == n
    assert custom_objects["BridgeModule"] is BridgeModule


def test_softmax_activation_shape_and_other_activations_unchanged():
    from deepctr_b200 import engine as E
    from deepctr_b200.layers import Activation
    E.clear_session()
    x = E.Input(shape=(7,), name="x")
    assert Activation("softmax")(x).shape == (None, 7)
    with pytest.raises(ValueError, match=r"unsupported activation 'elu' \(relu, sigmoid, tanh, linear, dice\)"):
        Activation("elu")


@pytest.mark.parametrize("bridge_type", BRIDGES)
def test_planner_fuses_the_gates_and_the_inner_bridges(bridge_type):
    """Layer 0's two gates are one launch on the embeddings; each inner boundary is one launch: the bridge with both
    gates, or, for 'concatenation', both gates on the bridge Dense's reshaped output."""
    model = _edcn(_columns(), cross_num=3, bridge_type=bridge_type)
    plan = model.planner.regulate_plan
    if bridge_type == "concatenation":
        assert len(plan.pairs) == 3 and not plan.bridges
    else:
        assert len(plan.pairs) == 1 and len(plan.bridges) == 2


def test_other_builders_plan_no_regulation():
    from deepctr_b200 import engine as E, models as M
    cols = _columns()
    for b in ("DeepFM", "DCN", "PNN"):
        E.clear_session()
        m = getattr(M, b)(cols, cols) if b != "PNN" else M.PNN(cols)
        assert not m.planner.regulate_plan.pairs and not m.planner.regulate_plan.bridges, b


def test_regulate_descriptor_layout_matches_header():
    from deepctr_b200 import _lib as L
    assert ctypes.sizeof(L.Regulate) == 264
    assert L.Regulate.u.offset == 112 and L.Regulate.dg1.offset == 256
