"""CPU: FwFM / DeepFEFM and their layers (FwFMLayer, FEFMLayer) against fixtures the reference's own layer and builder
code produced (tests/golden/generate_fefm.py):

1. the CPU restatement of tests/fefm_oracle.py (built on oracle/) reproduces every layer output and, with the
   checks shared by every family (model_golden_checks), every model fixture, weight set, graph and keyword default;
2. the deepctr_b200 builders hold only what is reachable from the output;
3. the reference's build-time checks and messages, the documented kernel limits (ValueError) and DeepFEFM's
   NotImplementedError branch;
4. the placement of DeepFEFM's FEFM scores in the DNN input is planned for DeepFEFM's graph, and only there.
"""
import itertools

import numpy as np
import pytest

import golden_models as G
import model_golden_checks as C

T = C.model_tests("fefm")
test_oracle_matches_reference_model = T.oracle
test_builder_creates_the_reference_weight_set = T.weight_set
test_builder_graph_is_the_reference_graph = T.graph
test_reference_default_arguments_are_the_same = T.defaults
L = C.layer_tests("fefm")
test_oracle_matches_reference_layer = L.oracle


def test_fixture_sets():
    C.check_fixture_set(G.FAMILIES["fefm"])
    L.fixture_set()
    ls = G.LAYER_SETS["fefm"]
    for name in ls.cases:
        meta, d = ls.load(name)
        if meta["layer"] == "FwFMLayer":
            g = d["g_field_pair_strengths"]
            assert not np.any(np.tril(g)), "the strengths' gradient is 0 on and below the diagonal"


def test_unreachable_branches_hold_no_weights():
    """With dnn_hidden_units=() the reference still creates a DNN and a Dense(1) (and, without use_linear, the
    linear part); they are off the output path, so neither graph holds them."""
    fam = G.FAMILIES["fefm"]
    model = G.build(fam.fixture("deepfefm_linear_fefm"))
    assert not any(type(l).__name__ in ("DNN", "Dense") for l in model.layers)
    assert not any("dense" in w.name or w.name.startswith("dnn") for w in model.weights)
    model = G.build(fam.fixture("deepfefm_no_linear"))
    assert not any(w.name.startswith("linear") for w in model.weights)


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
