"""TEST INFRASTRUCTURE - the FLEN fixture families (tests/golden/models_flen and tests/golden/flen, written by
tests/golden/generate_flen.py): how a model fixture's weights map onto tests/flen_oracle.py, how a layer fixture's
inputs reach the layer, and their records in golden_models.FAMILIES and golden_models.LAYER_SETS, added when this
module is imported so that model_golden_checks.model_tests("flen"), gpu_model_tests("flen"), layer_tests("flen")
and gpu_layer_test("flen") find them."""
import numpy as np
import torch

import golden_models as G


def flen_weights(fx, requires_grad=False):
    """golden_models.oracle_weights plus W['fwbi'] (the layer's kernel_mf, kernel_fm, bias_mf, bias_fm) and
    W['dnn_bn']."""
    W, leaves = G.oracle_weights(fx, requires_grad)

    def t(key):
        return G._leaf(fx, leaves, key, requires_grad) if key in fx.w else None

    (n,) = fx.layer_names("FieldWiseBiInteraction")
    W["fwbi"] = [t("%s/%s" % (n, w)) for w in ("kernel_mf", "kernel_fm", "bias_mf", "bias_fm")]
    W["dnn_bn"] = None
    for d in fx.layer_names("DNN"):
        k = len(W.get("dnn_kernels", []))
        if "%s/bn0/gamma" % d in fx.w:
            W["dnn_bn"] = [{p: t("%s/bn%d/%s" % (d, i, p)) for p in ("gamma", "beta")} for i in range(k)]
    return W, leaves


def flen_forward(fx, W):
    import flen_oracle as FO
    from deepctr_b200 import feature_column as FC
    return FO.flen(fx.inputs(), G.columns(fx, "linear", FC), G.columns(fx, "dnn", FC), W, task=fx.task)


def _flen_layer(meta, xs, W, d):
    import flen_oracle as FO
    return FO.field_wise_bi(xs, W["kernel_mf"], W["kernel_fm"], W.get("bias_mf"), W.get("bias_fm"))


def _flen_args(meta, d, device):
    """The groups as a model hands them over: windows of one wider [B, ld] buffer, in reverse order and one column
    apart (not adjacent, not 16-byte aligned), read in place; the buffer collects ``gx_<g>``."""
    from deepctr_b200 import engine as E, ops
    keys = G.numbered(d, "x_")
    xs = [d[k] for k in keys]
    b = xs[0].shape[0]
    widths = [int(np.prod(x.shape[1:])) for x in xs]
    col, cols = 1, {}
    for k, w in reversed(list(zip(keys, widths))):
        cols[k] = col
        col += w + 1
    buf = torch.zeros((b, col), dtype=torch.float32, device=device)
    for k, x, w in zip(keys, xs, widths):
        buf[:, cols[k]:cols[k] + w] = torch.tensor(x.reshape(b, w), device=device)
    base = E.Var(buf, requires_grad=True)
    return ([ops._window(base, cols[k], w, x.shape) for k, x, w in zip(keys, xs, widths)],
            {k: _Cols(base, cols[k], w) for k, w in zip(keys, widths)})


class _Cols(object):
    """The gradient of a window's columns of a buffer Var (what the layer test compares with ``gx_<g>``)."""

    def __init__(self, base, col0, w):
        self.base, self.col0, self.w = base, col0, w

    @property
    def grad(self):
        g = self.base.grad
        return g[:, self.col0:self.col0 + self.w] if g is not None else None


FAMILY = G.Family("models_flen", "reference_builders_flen.json", ("FLEN",), flen_weights, flen_forward, 12,
                  {"binary", "regression"},
                  # the embedding tables are created first; the graph reaches the linear tables first
                  graph_weight_order=("flen_contiguous", "flen_defaults", "flen_dnn_bn", "flen_eight_groups",
                                      "flen_hashed", "flen_no_dnn", "flen_reference_test", "flen_regression",
                                      "flen_run_flen_layout", "flen_two_groups", "flen_unequal_groups",
                                      "flen_varlen"))
G.FAMILIES.setdefault("flen", FAMILY)
G.LAYER_SETS.setdefault("flen", G.LayerSet("flen", 6, ("FieldWiseBiInteraction",), _flen_args, oracle=_flen_layer,
                                           cpu=G._FAMILY_CPU, gpu=(G._FAMILY_GPU, G._FAMILY_GPU)))
