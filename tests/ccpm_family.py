"""TEST INFRASTRUCTURE - the CCPM fixture families (tests/golden/models_ccpm and tests/golden/ccpm, written by
tests/golden/generate_ccpm.py): how a model fixture's weights map onto tests/ccpm_oracle.py, how a layer fixture's
input reaches the layer, and their records in golden_models.FAMILIES and golden_models.LAYER_SETS, added when this
module is imported so that model_golden_checks.model_tests("ccpm"), gpu_model_tests("ccpm"), layer_tests("ccpm")
and gpu_layer_test("ccpm") find them."""
import numpy as np
import torch

import golden_models as G


def ccpm_weights(fx, requires_grad=False):
    """golden_models.oracle_weights plus W['conv'], the Conv2D (kernel, bias) pairs in creation order."""
    W, leaves = G.oracle_weights(fx, requires_grad)
    W["conv"] = [(G._leaf(fx, leaves, n + "/kernel", requires_grad), G._leaf(fx, leaves, n + "/bias", requires_grad))
                 for n in sorted(fx.layer_names("Conv2D"), key=G._creation_order)]
    return W, leaves


def ccpm_forward(fx, W):
    import ccpm_oracle as CO
    from deepctr_b200 import feature_column as FC
    kw = fx.kwargs
    return CO.ccpm(fx.inputs(), G.columns(fx, "linear", FC), G.columns(fx, "dnn", FC), W,
                   conv_kernel_width=tuple(kw.get("conv_kernel_width", (6, 5))),
                   conv_filters=tuple(kw.get("conv_filters", (4, 4))), task=fx.task)


def _ccpm_layer(meta, xs, W, d):
    import ccpm_oracle as CO
    kw = meta["kwargs"]
    if meta["layer"] == "Conv2D":
        return CO.conv2d(xs[0], W["kernel"], W.get("bias"), kw.get("activation"))
    return CO.kmax(xs[0], kw["k"], kw["axis"])


def _ccpm_args(meta, d, device):
    """``x`` as a model hands it over: a window of a wider [B, ld] buffer read in place; the buffer collects ``gx``."""
    from deepctr_b200 import engine as E, ops
    x = d["x"]
    b, w = x.shape[0], int(np.prod(x.shape[1:]))
    buf = torch.zeros((b, w + 3), dtype=torch.float32, device=device)
    buf[:, 1:1 + w] = torch.tensor(x.reshape(b, w), device=device)
    base = E.Var(buf, requires_grad=True)
    return ops._window(base, 1, w, x.shape), {"x": _Cols(base, 1, w)}


class _Cols(object):
    """The gradient of the window's columns of a buffer Var (what the layer test compares with ``gx``)."""

    def __init__(self, base, col0, w):
        self.base, self.col0, self.w = base, col0, w

    @property
    def grad(self):
        g = self.base.grad
        return g[:, self.col0:self.col0 + self.w] if g is not None else None


FAMILY = G.Family("models_ccpm", "reference_builders_ccpm.json", ("CCPM",), ccpm_weights, ccpm_forward, 11,
                  {"binary", "regression"},
                  # the linear tables are created first; the graph reaches them after the convolution stack
                  graph_weight_order=("ccpm_defaults", "ccpm_dense_linear_only", "ccpm_hashed_varlen", "ccpm_no_conv",
                                      "ccpm_no_dnn", "ccpm_one_layer", "ccpm_reference_test", "ccpm_regression",
                                      "ccpm_three_layers", "ccpm_two_fields", "ccpm_wide_kernel"))
G.FAMILIES.setdefault("ccpm", FAMILY)
G.LAYER_SETS.setdefault("ccpm", G.LayerSet("ccpm", 7, ("Conv2D", "KMaxPooling"), _ccpm_args, oracle=_ccpm_layer,
                                           cpu=G._FAMILY_CPU, gpu=(G._FAMILY_GPU, G._FAMILY_GPU)))
