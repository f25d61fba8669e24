"""CPU: CCPM against fixtures the reference's own builder, layer and feature-column code produced
(tests/golden/generate_ccpm.py): the model fixtures, weight sets, graphs and keyword defaults with the checks shared
by every family (model_golden_checks), the Conv2D / KMaxPooling layer fixtures against the CPU restatement, the
reference's build-time errors and this package's deviations and limits, the k schedule, the planner's fused
convolution stack and the descriptor layout of b2ctr_conv_stack.
"""
import ctypes

import pytest

import model_golden_checks as C
import ccpm_family  # noqa: F401  (registers the "ccpm" fixture families)

T = C.model_tests("ccpm")
test_oracle_matches_reference_model = T.oracle
test_builder_creates_the_reference_weight_set = T.weight_set
test_builder_graph_is_the_reference_graph = T.graph
test_reference_default_arguments_are_the_same = T.defaults
test_fixture_set = T.fixture_set
LT = C.layer_tests("ccpm")
test_oracle_matches_reference_layer = LT.oracle
test_layer_fixture_set = LT.fixture_set


def _columns(n_sparse=4, dim=4, dense=False):
    from deepctr_b200 import feature_column as FC
    cols = [FC.SparseFeat("C%d" % i, 30, dim) for i in range(n_sparse)]
    return cols + ([FC.DenseFeat("I0", 1)] if dense else [])


def _ccpm(cols, linear=None, **kw):
    from deepctr_b200 import engine as E, models as M
    E.clear_session()
    return M.CCPM(cols if linear is None else linear, cols, **kw)


def test_mismatched_widths_and_filters_raise_the_reference_error():
    with pytest.raises(ValueError, match="conv_kernel_width must have same element with conv_filters"):
        _ccpm(_columns(), conv_kernel_width=(3,), conv_filters=(2, 2))


def test_dense_feature_in_dnn_columns_is_rejected_and_legal_in_linear_columns():
    with pytest.raises(ValueError, match="DenseFeat is not supported in dnn_feature_columns"):
        _ccpm(_columns(dense=True))
    m = _ccpm(_columns(), linear=_columns(dense=True))
    assert "I0" in m.input_names


def test_mismatched_embedding_dims_are_a_build_time_error():
    from deepctr_b200 import feature_column as FC
    cols = [FC.SparseFeat("a", 10, 4), FC.SparseFeat("b", 10, 8)]
    with pytest.raises(ValueError, match="embedding dimensions 4 and 8"):
        _ccpm(cols)


def _kmax(k, axis, shape):
    from deepctr_b200 import engine as E
    from deepctr_b200.layers import KMaxPooling
    E.clear_session()
    return KMaxPooling(k=k, axis=axis)(E.Input(shape=shape, name="x"))


@pytest.mark.parametrize("k,axis,msg", [(1, 0, r"axis must be 1~4,now is 0"), (1, -1, r"axis must be 1~4,now is -1"),
                                        (0, 1, r"k must be in 1 ~ 10,now k is 0"),
                                        (11, 1, r"k must be in 1 ~ 10,now k is 11"),
                                        (3, 4, r"axis must be 1~3,now is 4: axis 4 is past the last axis")])
def test_kmax_pooling_build_errors(k, axis, msg):
    with pytest.raises(ValueError, match=msg):
        _kmax(k, axis, (10, 4, 2))


def test_kmax_pooling_shape_config_and_custom_objects():
    from deepctr_b200.layers import KMaxPooling, custom_objects
    assert _kmax(3, 2, (4, 10, 2)).shape == (None, 4, 3, 2)
    assert KMaxPooling(k=3, axis=1).get_config()["k"] == 3
    assert custom_objects["KMaxPooling"] is KMaxPooling


@pytest.mark.parametrize("kw,arg", [(dict(kernel_size=(3, 3)), "kernel_size"), (dict(strides=(2, 1)), "strides"),
                                    (dict(padding="valid"), "padding"),
                                    (dict(data_format="channels_first"), "data_format"),
                                    (dict(dilation_rate=(2, 1)), "dilation_rate"), (dict(activation="dice"), "activation")])
def test_conv2d_configurations_ccpm_does_not_use_raise(kw, arg):
    from deepctr_b200.layers import Conv2D
    args = dict(filters=2, kernel_size=(3, 1), strides=(1, 1), padding="same")
    args.update(kw)
    with pytest.raises(NotImplementedError, match="Conv2D %s" % arg):
        Conv2D(**args)


def test_conv2d_weights_shape_and_defaults():
    import numpy as np
    from deepctr_b200 import engine as E
    from deepctr_b200.layers import Conv2D
    E.clear_session()
    conv = Conv2D(filters=4, kernel_size=(6, 1), strides=(1, 1), padding='same', activation='tanh', use_bias=True)
    y = conv(E.Input(shape=(26, 8, 1), name="x"))
    assert y.shape == (None, 26, 8, 4)
    assert [(w.name, w.shape) for w in conv.weights] == [("conv2d/kernel", (6, 1, 1, 4)), ("conv2d/bias", (4,))]
    k = conv.kernel.value()
    lim = np.sqrt(6.0 / (6 * 1 + 6 * 4))                 # glorot_uniform, fans over the receptive field
    assert np.abs(k).max() <= lim and np.abs(k).max() > 0.5 * lim
    np.testing.assert_array_equal(conv.bias.value(), 0)


@pytest.mark.parametrize("shape,kw,limit", [((65, 4, 1), dict(filters=2, kernel_size=(3, 1)), "CONV_MAX_ROWS"),
                                            ((26, 4, 1), dict(filters=17, kernel_size=(3, 1)), "CONV_MAX_CHANNELS"),
                                            ((26, 4, 1), dict(filters=2, kernel_size=(33, 1)), "CONV_MAX_WIDTH"),
                                            ((64, 4, 8), dict(filters=8, kernel_size=(3, 1)), "CONV_SMEM_BYTES")])
def test_conv2d_limits_raise_naming_them(shape, kw, limit):
    from deepctr_b200 import engine as E
    from deepctr_b200.layers import Conv2D
    E.clear_session()
    with pytest.raises(ValueError, match=limit):
        Conv2D(padding="same", **kw)(E.Input(shape=shape, name="x"))


def test_reference_default_shapes_are_inside_the_limits():
    """The defaults at 26 and 39 fields with E up to 64 build, and the planner fuses them."""
    for n in (26, 39):
        for dim in (4, 64):
            m = _ccpm(_columns(n, dim))
            assert len(m.planner.conv_plan.chains) == 1


def _schedule(l, n):
    """ccpm.py:62-69 restated: the k of each layer after the clamp to the rows it pools."""
    rows, ks = n, []
    for i in range(1, l + 1):
        k = max(1, int((1 - pow(i / l, l - i)) * n)) if i < l else 3
        rows = min(k, rows)
        ks.append(rows)
    return ks


def test_k_schedule():
    from deepctr_b200.models.ccpm import ccpm_k
    assert _schedule(2, 26) == [13, 3] and _schedule(3, 10) == [8, 3, 3] and _schedule(2, 2) == [1, 1]
    for l in range(1, 6):
        for n in range(1, 65):
            rows, ks = n, []
            for i in range(1, l + 1):
                rows = min(ccpm_k(i, l, n), rows)
                ks.append(rows)
            assert ks == _schedule(l, n), (l, n)


@pytest.mark.parametrize("l", [1, 2, 3, 4, 5])
def test_built_models_follow_the_k_schedule(l):
    from deepctr_b200.layers import KMaxPooling
    for n in (1, 2, 3, 7, 26, 64):
        m = _ccpm(_columns(n), conv_kernel_width=(3,) * l, conv_filters=(2,) * l, dnn_hidden_units=(8,))
        assert [ly.k for ly in m.layers if isinstance(ly, KMaxPooling)] == _schedule(l, n), (l, n)


def test_planner_fuses_the_whole_stack():
    from deepctr_b200 import engine as E
    from deepctr_b200.layers import KMaxPooling
    m = _ccpm(_columns(6), conv_kernel_width=(4, 3, 2), conv_filters=(3, 2, 2))
    (chain,) = m.planner.conv_plan.chains.values()
    assert [type(n.layer) for n in chain] == [E.Conv2D, KMaxPooling] * 3
    m = _ccpm(_columns(6), conv_kernel_width=(), conv_filters=())
    assert not m.planner.conv_plan.chains


def test_other_builders_plan_no_convolution_stack():
    from deepctr_b200 import engine as E, models as M
    cols = _columns()
    for b in ("DeepFM", "PNN", "EDCN"):
        E.clear_session()
        m = M.PNN(cols) if b == "PNN" else getattr(M, b)(cols, cols)
        assert not m.planner.conv_plan.chains, b


def test_a_conv_output_with_a_second_consumer_is_not_fused():
    from deepctr_b200 import backend, engine as E
    from deepctr_b200.layers import KMaxPooling, concat_func
    E.clear_session()
    x = E.Input(shape=(6, 4), name="x")
    h = E.Lambda(lambda t: backend.expand_dims(t, axis=3))(concat_func([x]))
    c = E.Conv2D(2, (3, 1), padding="same", activation="tanh")(h)
    p = E.Flatten()(KMaxPooling(k=3, axis=1)(c))
    out = E.Dense(1)(E.Concatenate()([p, E.Flatten()(c)]))
    m = E.Model(inputs=[x], outputs=out)
    assert not m.planner.conv_plan.chains


def test_conv_stack_descriptor_layout_matches_header():
    from deepctr_b200 import _lib as L
    assert ctypes.sizeof(L.ConvStage) == 56 and L.ConvStage.kernel.offset == 24
    assert ctypes.sizeof(L.ConvStack) == 552
    assert L.ConvStack.batch.offset == 24 and L.ConvStack.out.offset == 56 and L.ConvStack.stage.offset == 104
