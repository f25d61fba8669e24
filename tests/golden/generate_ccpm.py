#!/usr/bin/env python
"""Generate the CCPM fixtures (the builder, and its Conv2D and KMaxPooling layers) from the REFERENCE's own,
unmodified deepctr/feature_column.py, deepctr/inputs.py, deepctr/layers/* (KMaxPooling in sequence.py) and
deepctr/models/ccpm.py, executed eagerly under the torch-backed ``tensorflow`` stand-in of tf_torch_shim.py (the
recipe of generate_onn.py and generate_edcn.py).

    python tests/golden/generate_ccpm.py          (build container only: needs the reference checkout)

The symbols CCPM needs beyond the shim are supplied here, so that tf_torch_shim.py and the other generators (and
with them every existing fixture) stay as they are:
  * ``tensorflow.keras.layers.Conv2D``: channels_last, strides (1, 1), padding 'same' as TF pads it - explicitly,
    (w - 1) // 2 rows before and the rest after - then torch.nn.functional.conv2d, a bias and the activation;
  * ``tf.nn.top_k``: a stable descending sort, which gives TF's rule that equal values keep the lower index first;
  * ``tf.expand_dims`` and ``tf.transpose`` are the shim's (torch's unsqueeze and permute).
Every top_k call checks the margin of its selection: in every pooled column, consecutive values of the sorted
order down to the (k+1)-th differ by at least 1e-4 relative at the selection boundary and 1e-5 among the selected,
so that a reordered fp32 sum cannot flip a selection or its order.  A fixture that misses it is drawn again with
the next seed.  For the graphs built from the reference's ccpm.py on this package, generate_builders._aliased is
given the package's Conv2D, Lambda and ``tensorflow.expand_dims``.

The reference's own tests/models/CCPM_test.py returns before building anything under TensorFlow 2, so these
fixtures are the only executed record of the reference's CCPM.

Writes
  tests/golden/ccpm/*.npz                   layer level: ``meta``, the input ``x``, every weight ``w_<name>``, the
                                            output ``out``, an upstream gradient ``dout`` and the gradients ``gx`` /
                                            ``g_<name>``;
  tests/golden/models_ccpm/*.npz            model level, the layout of tests/golden/models/;
  tests/golden/reference_builders_ccpm.json the graphs the reference's ccpm.py SOURCE FILE builds on this package
                                            for those fixtures, and its keyword defaults.
The existing fixture directories and JSON files are not touched.
"""
import importlib
import inspect
import json
import os
import shutil
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))

import tf_torch_shim as S  # noqa: E402
import generate_fefm as GF  # noqa: E402
import generate_pairwise as GP  # noqa: E402
from generate_models import _col_meta  # noqa: E402

REF = GF.REF
LAYER_OUT = os.path.join(HERE, "ccpm")
MODEL_OUT = os.path.join(HERE, "models_ccpm")
BUILDERS_JSON = os.path.join(HERE, "reference_builders_ccpm.json")
FILES = {"CCPM": ("models/ccpm.py", "models.ccpm")}
MARGIN_BOUNDARY, MARGIN_INSIDE = 1e-4, 1e-5
_SHORT = []          # selections of the current case that miss the margin


class Conv2D(S.Layer):
    """tf.keras.layers.Conv2D(filters, kernel_size, strides=(1, 1), padding='same', activation, use_bias)."""

    def __init__(self, filters, kernel_size, strides=(1, 1), padding="valid", activation=None, use_bias=True, **kw):
        S.Layer.__init__(self, name=kw.get("name"))
        assert tuple(strides) == (1, 1) and padding == "same", (strides, padding)
        self.filters, self.kernel_size = int(filters), tuple(int(k) for k in kernel_size)
        self.activation, self.use_bias = activation, use_bias

    def build(self, input_shape):
        kh, kw = self.kernel_size
        self.kernel = self.add_weight(name="kernel", shape=(kh, kw, int(input_shape[-1]), self.filters))
        self.bias = self.add_weight(name="bias", shape=(self.filters,)) if self.use_bias else None
        self.built = True

    def call(self, x, **kw):
        kh, kwd = self.kernel_size
        # TF 'same': (k - 1) // 2 before, the rest after, per spatial axis
        pad = ((kwd - 1) // 2, kwd - 1 - (kwd - 1) // 2, (kh - 1) // 2, kh - 1 - (kh - 1) // 2)
        xp = torch.nn.functional.pad(x.permute(0, 3, 1, 2), pad)
        y = torch.nn.functional.conv2d(xp, self.kernel.permute(3, 2, 0, 1)).permute(0, 2, 3, 1)
        if self.bias is not None:
            y = y + self.bias
        return {None: lambda v: v, "linear": lambda v: v, "relu": torch.relu, "sigmoid": torch.sigmoid,
                "tanh": torch.tanh}[self.activation](y)


def _top_k(x, k=1, sorted=True, name=None):
    """tf.nn.top_k over the last axis: a stable descending sort; records a selection short of the margin."""
    vals, idx = torch.sort(x, dim=-1, descending=True, stable=True)
    v = vals.detach().numpy()
    n = v.shape[-1]
    top = v[..., :min(k + 1, n)]
    gap = np.abs(top[..., :-1] - top[..., 1:])
    scale = np.maximum(np.abs(top[..., :-1]), np.abs(top[..., 1:]))
    need = np.full(gap.shape[-1], MARGIN_INSIDE)
    if k < n:
        need[-1] = MARGIN_BOUNDARY
    if gap.size and np.any(gap < need * scale):
        _SHORT.append(float((gap / np.maximum(scale, 1e-30)).min()))
    return vals[..., :k], idx[..., :k]


def _install():
    S.install(REF)
    sys.modules["tensorflow.keras.layers"].Conv2D = Conv2D
    sys.modules["tensorflow"].nn.top_k = _top_k
    importlib.import_module("deepctr.feature_column")


def _retry(make, seed):
    """make(seed) until no selection misses the margin (the next seed each time)."""
    for s in range(seed, seed + 50):
        del _SHORT[:]
        make(s)
        if not _SHORT:
            return s
    raise AssertionError("no seed in [%d, %d) gives every selection its margin" % (seed, seed + 50))


def layer_case(name, cls, kwargs, shape, seed):
    def make(s):
        S.CTX.reset()
        S.CTX.rng = np.random.RandomState(s)
        S.CTX.grad = True
        rng = np.random.RandomState(s + 1000)
        x = rng.normal(0, 0.5, size=shape).astype(np.float32)
        xt = torch.tensor(x, requires_grad=True)
        if cls == "Conv2D":
            layer = Conv2D(**kwargs)
        else:
            layer = getattr(sys.modules["deepctr.layers.sequence"], cls)(**kwargs)
        out = layer(xt)
        dout = rng.normal(0, 1.0, size=tuple(out.shape)).astype(np.float32)
        leaves = [t for _, t in layer._w]
        grads = torch.autograd.grad((out * torch.as_tensor(dout)).sum(), [xt] + leaves)
        d = {"meta": np.array(json.dumps({"layer": cls, "kwargs": kwargs})), "x": x,
             "out": out.detach().numpy(), "dout": dout, "gx": grads[0].numpy()}
        for (wn, t), g in zip(layer._w, grads[1:]):
            d["w_" + wn] = t.detach().numpy().copy()
            d["g_" + wn] = g.numpy()
        np.savez_compressed(os.path.join(LAYER_OUT, name + ".npz"), **d)
        print("%-28s out%s  %d weights  seed %d" % (name, tuple(d["out"].shape), len(layer._w), s))
    _retry(make, seed)


def _cols(make_lin, make_dnn, kw):
    def f(FC):
        lin, dnn = make_lin(FC), make_dnn(FC)
        return (lin, dnn), dict(kw), {"linear": [_col_meta(c, FC) for c in lin],
                                      "dnn": [_col_meta(c, FC) for c in dnn]}
    return f


def model_case(name, make_lin, make_dnn, x, y, kw, seed, task="binary"):
    kw = dict(kw, l2_reg_linear=0, l2_reg_embedding=0)
    _retry(lambda s: GF.model_case(name, "CCPM", _cols(make_lin, make_dnn, kw), x, y, s, task=task), seed)


def _sparse(n_sparse, dim, vocab0=20):
    return lambda FC: [FC.SparseFeat("C%d" % (i + 1), vocab0 + 3 * i, dim) for i in range(n_sparse)]


def _ids(rng, n, n_sparse, vocab0=20):
    return {"C%d" % (i + 1): rng.randint(0, vocab0 + 3 * i, size=n).astype(np.int32) for i in range(n_sparse)}


def fixtures():
    _install()
    GF.MODULES["CCPM"] = "deepctr.models.ccpm"
    GF.MODEL_OUT = MODEL_OUT
    for d in (LAYER_OUT, MODEL_OUT):
        if os.path.isdir(d):
            shutil.rmtree(d)
        os.makedirs(d)

    # ---- layers: KMaxPooling at the reference test's shape (B, T, E, 2), k = 3, on axes 1, 2 and 3; Conv2D with
    #      widths 1, 5, 6, one and four input channels, tanh and linear
    layer_case("kmax_axis1", "KMaxPooling", dict(k=3, axis=1), (6, 10, 4, 2), 1)
    layer_case("kmax_axis2", "KMaxPooling", dict(k=3, axis=2), (6, 4, 10, 2), 2)
    layer_case("kmax_axis3", "KMaxPooling", dict(k=3, axis=3), (6, 4, 2, 10), 3)
    for w, cin, act, sd in ((1, 1, "tanh", 4), (5, 4, "linear", 5), (6, 1, "tanh", 6), (6, 4, "linear", 7)):
        layer_case("conv_w%d_c%d_%s" % (w, cin, act), "Conv2D",
                   dict(filters=3, kernel_size=(w, 1), strides=(1, 1), padding="same", activation=act,
                        use_bias=True), (5, 9, 4, cin), sd)

    rng = np.random.RandomState(20261022)
    n = 16
    y = lambda: (rng.rand(n) < 0.3).astype(np.float32)  # noqa: E731
    # ---- the defaults at 6 fields --------------------------------------------------------------------------
    x6 = _ids(rng, n, 6)
    model_case("ccpm_defaults", _sparse(6, 4), _sparse(6, 4), x6, y(), {}, 101)
    # ---- the reference test's configuration: 3 fields and a pooled varlen field ---------------------------
    T = 4
    lens = rng.randint(1, T + 1, size=n)
    seq = rng.randint(1, 13, size=(n, T)).astype(np.int32)
    seq[np.arange(T)[None, :] >= lens[:, None]] = 0
    x3 = dict(_ids(rng, n, 3), S1=seq)

    def varlen(FC):
        return _sparse(3, 4)(FC) + [FC.VarLenSparseFeat(FC.SparseFeat("S1", 13, 4), maxlen=T, combiner="mean")]
    ref_kw = dict(conv_kernel_width=(3, 2), conv_filters=(2, 1), dnn_hidden_units=(32,))
    model_case("ccpm_reference_test", varlen, varlen, x3, y(), ref_kw, 102)
    # ---- three layers at 10 fields (k = 8, 3, 3), one layer, no conv, 2 fields, width > fields ---------------
    x10 = _ids(rng, n, 10)
    model_case("ccpm_three_layers", _sparse(10, 4), _sparse(10, 4), x10, y(),
               dict(conv_kernel_width=(4, 3, 2), conv_filters=(3, 2, 2), dnn_hidden_units=(16,)), 103)
    model_case("ccpm_one_layer", _sparse(6, 4), _sparse(6, 4), x6, y(),
               dict(conv_kernel_width=(3,), conv_filters=(2,), dnn_hidden_units=(16,)), 104)
    model_case("ccpm_no_conv", _sparse(6, 4), _sparse(6, 4), x6, y(),
               dict(conv_kernel_width=(), conv_filters=(), dnn_hidden_units=(16,)), 105)
    x2 = _ids(rng, n, 2)
    model_case("ccpm_two_fields", _sparse(2, 4), _sparse(2, 4), x2, y(),
               dict(conv_kernel_width=(2, 2), conv_filters=(2, 2), dnn_hidden_units=(8,)), 106)
    x4 = _ids(rng, n, 4)
    model_case("ccpm_wide_kernel", _sparse(4, 4), _sparse(4, 4), x4, y(),
               dict(conv_kernel_width=(7, 6), conv_filters=(2, 2), dnn_hidden_units=(8,)), 107)
    # ---- no DNN, regression ----------------------------------------------------------------------------------
    model_case("ccpm_no_dnn", _sparse(6, 4), _sparse(6, 4), x6, y(), dict(dnn_hidden_units=()), 108)
    yr = rng.normal(0, 1, size=n).astype(np.float32)
    model_case("ccpm_regression", _sparse(6, 4), _sparse(6, 4), x6, yr, dict(dnn_hidden_units=(16,),
                                                                            task="regression"), 109,
               task="regression")
    # ---- hashed single-valued and varlen fields; a dense feature in the linear columns only -----------------
    xh = dict(_ids(rng, n, 3), h1=rng.randint(0, 1000, size=n).astype(np.int32),
              s_h=np.where(np.arange(T)[None, :] < lens[:, None], rng.randint(1, 1000, size=(n, T)), 0)
              .astype(np.int32))

    def hashed(FC):
        return _sparse(3, 4)(FC) + [FC.SparseFeat("h1", 7, 4, use_hash=True),
                                    FC.VarLenSparseFeat(FC.SparseFeat("s_h", 5, 4, use_hash=True), maxlen=T,
                                                        combiner="mean")]
    model_case("ccpm_hashed_varlen", hashed, hashed, xh, y(), dict(dnn_hidden_units=(8,)), 110)
    xd = dict(x6, I1=rng.rand(n).astype(np.float32))

    def with_dense(FC):
        return _sparse(6, 4)(FC) + [FC.DenseFeat("I1", 1)]
    model_case("ccpm_dense_linear_only", with_dense, _sparse(6, 4), xd, y(), dict(dnn_hidden_units=(8,)), 111)


def builders():
    import golden_models as G
    import generate_builders as GB
    from golden_models import signature, builder_args
    from deepctr_b200 import backend, engine as E
    from deepctr_b200.layers import sequence as SQ
    out = {"signatures": {}, "defaults": {}}
    names = sorted(os.path.basename(p)[:-4] for p in os.listdir(MODEL_OUT) if p.endswith(".npz"))
    GB._FILES.update(FILES)
    GP.MODEL_OUT = MODEL_OUT
    with GB._aliased():
        ly = sys.modules["tensorflow.keras.layers"]
        ly.Conv2D, ly.Lambda = E.Conv2D, E.Lambda
        sys.modules["tensorflow"].expand_dims = backend.expand_dims
        assert sys.modules["refdrop.layers.sequence"].KMaxPooling is SQ.KMaxPooling
        for name in names:
            fx = GP._fixture(name)
            args, kw = builder_args(fx)
            build = GB._reference_builder(os.path.join(REF, "deepctr"), fx.builder)
            E.clear_session()
            model = build(*args, **kw)
            G.weight_map(fx, model)
            out["signatures"][name] = signature(model)
        sig = inspect.signature(GB._reference_builder(os.path.join(REF, "deepctr"), "CCPM"))
        out["defaults"]["CCPM"] = [[k, repr(p.default)] for k, p in sig.parameters.items()]
    E.clear_session()
    with open(BUILDERS_JSON, "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
    print("wrote", os.path.basename(BUILDERS_JSON), sorted(out["signatures"]))


if __name__ == "__main__":
    fixtures()
    builders()
