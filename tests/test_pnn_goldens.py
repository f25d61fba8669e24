"""CPU: PNN and its layers (InnerProductLayer, OutterProductLayer) against fixtures the reference's own layer and
builder code produced (tests/golden/generate_pnn.py):

1. the CPU restatement of tests/pnn_oracle.py (built on oracle/) reproduces every layer output and, with the
   checks shared by every family (model_golden_checks), every model fixture, weight set, graph and keyword default;
2. the deepctr_b200 builder holds only what is reachable from the output;
3. the reference's checks and messages, the documented kernel limits (ValueError), get_config and Reshape;
4. the placement of PNN's products in the DNN input is planned for PNN's graph, and only there.
"""

import pytest

import golden_models as G
import model_golden_checks as C

T = C.model_tests("pnn")
test_oracle_matches_reference_model = T.oracle
test_builder_creates_the_reference_weight_set = T.weight_set
test_builder_graph_is_the_reference_graph = T.graph
test_reference_default_arguments_are_the_same = T.defaults
L = C.layer_tests("pnn")
test_oracle_matches_reference_layer = L.oracle


def test_fixture_sets():
    C.check_fixture_set(G.FAMILIES["pnn"])
    L.fixture_set()


def test_off_path_products_hold_no_weights():
    """The reference always builds and calls OutterProductLayer (and InnerProductLayer); the one a model does not
    use is off the output path, so the graph holds neither it nor its kernel."""
    for name, inner, outer in (("pnn_defaults", True, False), ("pnn_opnn_mat", False, True),
                               ("pnn_no_products", False, False), ("pnn_inner_outer_mat", True, True)):
        model = G.build(G.FAMILIES["pnn"].fixture(name))
        kinds = {type(l).__name__ for l in model.layers}
        assert ("InnerProductLayer" in kinds) == inner, name
        assert ("OutterProductLayer" in kinds) == outer, name
        assert any(w.name.endswith("/kernel") and "outter" in w.name for w in model.weights) == outer, name


def test_bad_kernel_type_raises():
    from deepctr_b200 import engine as E, models as M
    from deepctr_b200 import feature_column as FC
    from deepctr_b200.layers import OutterProductLayer
    cols = [FC.SparseFeat("C%d" % i, 30, 4) for i in range(4)]
    E.clear_session()
    with pytest.raises(ValueError) as e:
        M.PNN(cols, kernel_type="diag")
    assert str(e.value) == "kernel_type must be mat,vec or num"
    with pytest.raises(ValueError) as e:
        OutterProductLayer("diag")
    assert str(e.value) == "kernel_type must be mat,vec or num"


@pytest.mark.parametrize("nfields,dim", [(65, 4), (3, 65)])
def test_unsupported_shapes_raise(nfields, dim):
    from deepctr_b200 import engine as E
    from deepctr_b200.layers import InnerProductLayer, OutterProductLayer
    E.clear_session()
    shapes = [(None, 1, dim)] * nfields
    with pytest.raises(ValueError, match="InnerProductLayer supports 2 to 64 inputs and embedding_size 1 to 64"):
        InnerProductLayer().build(shapes)
    with pytest.raises(ValueError, match="OutterProductLayer supports 2 to 64 inputs and embedding_size 1 to 64"):
        OutterProductLayer("vec").build(shapes)


def test_layer_reference_checks_weights_and_config():
    from deepctr_b200 import engine as E
    from deepctr_b200.layers import InnerProductLayer, OutterProductLayer
    E.clear_session()
    for cls in (InnerProductLayer, OutterProductLayer):
        n = cls.__name__
        with pytest.raises(ValueError) as e:
            cls().build([(None, 1, 4)])
        assert str(e.value) == "A `%s` layer should be called on a list of at least 2 inputs" % n
        with pytest.raises(ValueError) as e:
            cls().build([(None, 1, 4), (None, 1, 8)])
        assert str(e.value).startswith("A `%s` layer requires inputs with same shapes Got different shapes: {" % n)
        with pytest.raises(ValueError) as e:
            cls().build([(None, 2, 4), (None, 2, 4)])
        assert str(e.value) == ("A `%s` layer requires inputs of a list with same shape tensor like "
                                "(None,1,embedding_size)Got different shapes: (None, 2, 4)" % n)
    E.clear_session()
    P = 6
    for kt, shape in (("mat", (5, P, 5)), ("vec", (P, 5)), ("num", (P, 1))):
        layer = OutterProductLayer(kt, seed=7)
        layer.build([(None, 1, 5)] * 4)
        assert [(w.name.split("/")[-1], w.shape) for w in layer.weights] == [("kernel", shape)]
        assert type(layer.kernel.initializer).__name__ == "GlorotUniform" and layer.kernel.initializer.seed == 7
        assert layer.compute_output_shape([(None, 1, 5)] * 4) == (None, P)
        cfg = layer.get_config()
        assert (cfg["kernel_type"], cfg["seed"]) == (kt, 7)
    inner = InnerProductLayer(reduce_sum=False)
    inner.build([(None, 1, 5)] * 4)
    assert inner.weights == []
    assert inner.compute_output_shape([(None, 1, 5)] * 4) == (None, P, 5)
    assert InnerProductLayer().compute_output_shape([(None, 1, 5)] * 4) == (None, P, 1)
    assert inner.get_config()["reduce_sum"] is False


def test_mat_kernel_fans_follow_keras():
    """glorot_uniform on the 3-D [E, P, E] kernel: Keras' fans (P*E, E*E), from engine._fans."""
    from deepctr_b200 import engine as E
    assert E._fans((5, 6, 5)) == (6 * 5, 5 * 5)


def test_reshape_layer():
    from deepctr_b200 import engine as E
    r = E.Reshape([12])
    assert r.compute_output_shape((None, 3, 4)) == (None, 12)
    assert E.Reshape((3, -1)).compute_output_shape((None, 12)) == (None, 3, 4)
    assert r.get_config()["target_shape"] == (12,)
    with pytest.raises(ValueError, match="total size of new array must be unchanged"):
        E.Reshape([5]).compute_output_shape((None, 3, 4))


def test_pnn_placement_is_planned_for_pnn_only():
    """PNN's products get their columns between the embeddings and the dense columns of the gather buffer when its DNN
    input is concat([linear_signal, products]) through combined_dnn_input; every other model keeps its row pitch."""
    from deepctr_b200 import engine as E, inputs as I, models as M
    from deepctr_b200 import feature_column as FC
    cols = [FC.SparseFeat("C%d" % i, 30, 8) for i in range(6)] + [FC.DenseFeat("I%d" % i, 1) for i in range(3)]

    def plan(model):
        p = model.planner
        return p.main_width, p.main_ld, p.pnn_cols, sorted(p.pnn_places.values())
    # 6 x 8 = 48 embedding columns + P = 15 per product + 3 dense, padded to 4
    for kw, want in ((dict(), (48, 68, 15, [0])),
                     (dict(use_inner=False, use_outter=True), (48, 68, 15, [0])),
                     (dict(use_outter=True), (48, 84, 30, [0, 15])),
                     (dict(use_outter=True, kernel_type="num"), (48, 84, 30, [0, 15])),
                     (dict(use_inner=False), (48, 52, 0, []))):
        E.clear_session()
        assert plan(M.PNN(cols, **kw)) == want, kw
    E.clear_session()
    assert plan(M.PNN(cols[:6], use_outter=True)) == (48, 80, 30, [0, 15])     # no dense features: 78 -> 80
    for builder in ("DeepFM", "NFM", "FiBiNET", "FwFM", "DeepFEFM"):
        E.clear_session()
        model = getattr(M, builder)(cols, cols)
        assert model.planner.pnn_places == {} and model.planner.pnn_cols == 0, builder
        assert model.planner.main_ld == (68 if builder == "DeepFEFM" else 52), builder
    I.DNN_INPUT_PLACEMENT = False
    try:
        E.clear_session()
        assert plan(M.PNN(cols, use_outter=True)) == (48, 52, 0, [])
    finally:
        I.DNN_INPUT_PLACEMENT = True
