"""CPU: FLEN against fixtures the reference's own builder, layer and feature-column code produced
(tests/golden/generate_flen.py): the model fixtures, weight sets, graphs and keyword defaults with the checks shared
by every family (model_golden_checks), the FieldWiseBiInteraction layer fixtures against the CPU restatement, the
reference's errors and this package's deviation and limits, what the planner claims and the descriptor layout of
b2ctr_field_wise_bi.
"""
import ctypes

import pytest

import model_golden_checks as C
import flen_family  # noqa: F401  (registers the "flen" fixture families)

T = C.model_tests("flen")
test_oracle_matches_reference_model = T.oracle
test_builder_creates_the_reference_weight_set = T.weight_set
test_builder_graph_is_the_reference_graph = T.graph
test_reference_default_arguments_are_the_same = T.defaults
test_fixture_set = T.fixture_set
LT = C.layer_tests("flen")
test_oracle_matches_reference_layer = LT.oracle
test_layer_fixture_set = LT.fixture_set


def _columns(groups, dim=4, dense=0):
    from deepctr_b200 import feature_column as FC
    cols = [FC.SparseFeat("C%d" % i, 30, dim, group_name=g) for i, g in enumerate(groups)]
    return cols + [FC.DenseFeat("I%d" % i, 1) for i in range(dense)]


def _flen(cols, **kw):
    from deepctr_b200 import engine as E, models as M
    E.clear_session()
    return M.FLEN(cols, cols, **kw)


def _layer(shapes, **kw):
    from deepctr_b200 import engine as E
    from deepctr_b200.layers import FieldWiseBiInteraction
    E.clear_session()
    layer = FieldWiseBiInteraction(**kw)
    return layer, layer([E.Input(shape=s, name="x%d" % i) for i, s in enumerate(shapes)])


def test_a_single_group_raises_the_reference_error():
    with pytest.raises(ValueError, match="should be called on a list of at least 2 inputs"):
        _flen(_columns(["a", "a", "a"]))
    with pytest.raises(ValueError, match="should be called on a list of at least 2 inputs"):
        _layer([(3, 4)])


def test_mismatched_embedding_dims_are_a_build_time_error():
    from deepctr_b200 import feature_column as FC
    cols = [FC.SparseFeat("a", 10, 4, group_name="u"), FC.SparseFeat("b", 10, 8, group_name="i")]
    with pytest.raises(ValueError, match="embedding dimensions 4 and 8"):
        _flen(cols)


@pytest.mark.parametrize("shapes,limit", [([(1, 4)] * 9, "FWBI_MAX_GROUPS"), ([(200, 4), (57, 4)], "FWBI_MAX_FIELDS"),
                                          ([(2, 257), (2, 257)], "FWBI_MAX_DIM")])
def test_shapes_outside_the_kernel_limits_raise_naming_the_limit(shapes, limit):
    with pytest.raises(ValueError, match=limit):
        _layer(shapes)


def test_layer_weights_initialisers_and_config():
    import numpy as np
    layer, out = _layer([(2, 4), (3, 4), (1, 4)])
    assert tuple(out.shape) == (None, 4) or tuple(out.shape)[1:] == (4,)
    w = {v.name.split("/", 1)[1]: v for v in layer.weights}
    assert sorted(w) == ["bias_fm", "bias_mf", "kernel_fm", "kernel_mf"]
    assert w["kernel_mf"].shape == (3, 1) and w["kernel_fm"].shape == (3, 1) and w["bias_mf"].shape == (4,)
    np.testing.assert_array_equal(w["kernel_mf"].value(), 1.0)
    np.testing.assert_array_equal(w["kernel_fm"].value(), 0.5)
    np.testing.assert_array_equal(w["bias_fm"].value(), 0.0)
    cfg = layer.get_config()
    assert cfg["use_bias"] is True and cfg["seed"] == 1024
    layer, _ = _layer([(2, 4), (3, 4)], use_bias=False, seed=7)
    assert sorted(v.name.split("/", 1)[1] for v in layer.weights) == ["kernel_fm", "kernel_mf"]
    assert layer.get_config()["seed"] == 7
    from deepctr_b200.layers import custom_objects
    assert custom_objects["FieldWiseBiInteraction"] is type(layer)


def _plan(model):
    return model.planner.field_wise_plan


def test_planner_claims_flen_with_interleaved_and_one_member_groups():
    m = _flen(_columns(["a", "b", "c", "a", "b", "a"], dense=2), dnn_hidden_units=(8,))
    (groups,) = _plan(m).groups.values()
    assert [len(g) for g in groups] == [3, 2, 1]
    assert len(_plan(m).virtual) == 3
    assert sorted(type(n.layer).__name__ for n in _plan(m).virtual) == ["Concat", "Concat", "NoMask"]


def test_planner_leaves_a_concat_with_a_second_consumer():
    from deepctr_b200 import engine as E
    from deepctr_b200.feature_column import build_input_features, input_from_feature_columns
    from deepctr_b200.layers import FieldWiseBiInteraction, concat_func, PredictionLayer
    E.clear_session()
    cols = _columns(["a", "b", "a", "b"])
    feats = build_input_features(cols)
    groups, _ = input_from_feature_columns(feats, cols, 0, 1024, support_group=True)
    cats = [concat_func(v, axis=1) for v in groups.values()]
    h = FieldWiseBiInteraction()(cats)
    extra = E.Flatten()(cats[0])
    out = PredictionLayer()(E.Dense(1)(concat_func([h, extra])))
    m = E.Model(inputs=list(feats.values()), outputs=out)
    assert not _plan(m).groups and not _plan(m).virtual


def test_planner_leaves_a_layer_called_twice_and_a_non_window_input():
    from deepctr_b200 import engine as E
    from deepctr_b200.feature_column import build_input_features, input_from_feature_columns
    from deepctr_b200.layers import FieldWiseBiInteraction, concat_func, PredictionLayer
    cols = _columns(["a", "b", "a", "b"])
    for case in ("twice", "non_window"):
        E.clear_session()
        feats = build_input_features(cols)
        groups, _ = input_from_feature_columns(feats, cols, 0, 1024, support_group=True)
        vs = list(groups.values())
        layer = FieldWiseBiInteraction()
        if case == "twice":
            h1 = layer([concat_func(v, axis=1) for v in vs])
            h2 = layer([concat_func(v, axis=1) for v in vs])
            h = concat_func([h1, h2])
        else:
            scaled = E.Lambda(lambda t: t)(concat_func(vs[0], axis=1))
            h = layer([scaled, concat_func(vs[1], axis=1)])
        out = PredictionLayer()(E.Dense(1)(h))
        m = E.Model(inputs=list(feats.values()), outputs=out)
        assert not _plan(m).groups and not _plan(m).virtual, case


def test_field_wise_bi_descriptor_layout_matches_header():
    from deepctr_b200 import _lib as L
    S = L.FieldWiseBi
    assert L.FWBI_MAX_FIELDS == 256 and L.FWBI_MAX_GROUPS == 8
    assert ctypes.sizeof(S) == 3224
    assert S.batch.offset == 24 and S.col.offset == 48 and S.group.offset == 2096
    assert S.kernel_mf.offset == 3120 and S.out.offset == 3152 and S.dbias_fm.offset == 3216
