#!/usr/bin/env python
"""Generate the ONN fixtures from the REFERENCE's own, unmodified deepctr/feature_column.py, deepctr/inputs.py,
deepctr/layers/* and deepctr/models/onn.py, executed eagerly under the torch-backed ``tensorflow`` stand-in of
tf_torch_shim.py (the recipe of generate_pnn.py).

    python tests/golden/generate_onn.py          (build container only: needs the reference checkout)

The symbols ONN needs beyond the shim are supplied here, so that tf_torch_shim.py and generate_builders.py (and with
them every existing fixture) stay as they are:
  * ``tensorflow.keras.layers.multiply`` (the elementwise product of the shim's tensors);
  * ``tensorflow.keras.backend.sum``;
  * a full Keras ``BatchNormalization``: trainable ``gamma`` / ``beta`` and the non-trainable ``moving_mean`` /
    ``moving_variance``, named as Keras names them (the shim's has neither).
ONN's ``l2`` import path (tensorflow.keras.regularizers) is the shim's.  For the graphs built from the reference's
onn.py on this package, generate_builders._aliased is given the package's Embedding, Lambda, multiply,
BatchNormalization, backend and l2.

Training-mode BatchNormalization: the models run as train_on_batch runs them, normalising with the batch statistics.
The fixture stores those batch statistics as the moving statistics, so that a prediction (which normalises with the
moving statistics) gives the same logits: the forward check and the SGD-step check then compare against the same
recorded outputs, loss and gradients.  Dropout stays 0: Keras' dropout RNG is not pinned.

Writes
  tests/golden/models_onn/*.npz             model level, the layout of tests/golden/models/;
  tests/golden/reference_builders_onn.json  the graphs the reference's onn.py SOURCE FILE builds on this package for
                                            those fixtures, and its keyword defaults.
The existing fixture directories and JSON files are not touched.
"""
import importlib
import inspect
import json
import os
import shutil
import sys
import types

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
from generate_models import _col_meta, criteo_like  # noqa: E402

REF = GF.REF
MODEL_OUT = os.path.join(HERE, "models_onn")
BUILDERS_JSON = os.path.join(HERE, "reference_builders_onn.json")
FILES = {"ONN": ("models/onn.py", "models.onn")}


class BatchNormalization(S.Layer):
    """tf.keras.layers.BatchNormalization over the last axis, in training mode (batch statistics, biased variance,
    epsilon 1e-3).  The batch statistics are written into the moving statistics (see the module docstring)."""

    def __init__(self, axis=-1, momentum=0.99, epsilon=1e-3, center=True, scale=True, **kw):
        S.Layer.__init__(self, **kw)
        self.epsilon = epsilon

    def build(self, input_shape):
        n = int(input_shape[-1])
        self.gamma = self.add_weight(name="gamma", shape=(n,))
        with torch.no_grad():
            self.gamma.add_(1.0)                     # around Keras' ones
        self.beta = self.add_weight(name="beta", shape=(n,))
        self.moving_mean = self.add_weight(name="moving_mean", shape=(n,), trainable=False)
        self.moving_variance = self.add_weight(name="moving_variance", shape=(n,), trainable=False)
        self.built = True

    def call(self, x, training=None, **kwargs):
        red = tuple(range(x.dim() - 1))
        mean, var = x.mean(dim=red), x.var(dim=red, unbiased=False)
        with torch.no_grad():
            self.moving_mean.copy_(mean)
            self.moving_variance.copy_(var)
        return (x - mean) / torch.sqrt(var + self.epsilon) * self.gamma + self.beta


def _multiply(inputs, **kw):
    out = inputs[0]
    for t in inputs[1:]:
        out = out * t
    return out


def _install():
    S.install(REF)
    layers = sys.modules["tensorflow.keras.layers"]
    layers.multiply = _multiply
    layers.BatchNormalization = BatchNormalization
    sys.modules["tensorflow.keras.backend"].sum = lambda x, axis=None, keepdims=False: torch.sum(
        x, dim=axis, keepdim=keepdims)
    importlib.import_module("deepctr.feature_column")


def _varlen_case(rng, n=32, T=4, hashed=False):
    """Single-valued fields, a dense feature and pooled varlen fields with the combiners sum / mean / max (padding
    id 0 masked).  ``hashed``: one single-valued and one varlen column hashed on the fly; ONN's Hash keeps no id for
    padding, so the varlen mask is (hashed id != 0), not (raw id != 0)."""
    lens = rng.randint(1, T + 1, size=n).astype(np.int32)

    def padded(vocab):
        a = rng.randint(1, vocab, size=(n, T)).astype(np.int32)
        a[np.arange(T)[None, :] >= lens[:, None]] = 0
        return a
    x = {"C1": rng.randint(0, 20, size=n).astype(np.int32), "C2": rng.randint(0, 23, size=n).astype(np.int32),
         "I1": rng.rand(n).astype(np.float32)}
    if hashed:
        x["h1"] = rng.randint(0, 1000, size=n).astype(np.int32)
        x["s_h"] = padded(1000)
    else:
        x.update({"s_sum": padded(13), "s_mean": padded(15), "s_max": padded(11)})
    y = (rng.rand(n) < 0.3).astype(np.float32)

    def make(FC):
        cols = [FC.SparseFeat("C1", 20, 4), FC.SparseFeat("C2", 23, 4), FC.DenseFeat("I1", 1)]
        if hashed:
            cols += [FC.SparseFeat("h1", 7, 4, use_hash=True),
                     FC.VarLenSparseFeat(FC.SparseFeat("s_h", 5, 4, use_hash=True), maxlen=T, combiner="mean")]
        else:
            cols += [FC.VarLenSparseFeat(FC.SparseFeat("s_sum", 13, 4), maxlen=T, combiner="sum"),
                     FC.VarLenSparseFeat(FC.SparseFeat("s_mean", 15, 4), maxlen=T, combiner="mean"),
                     FC.VarLenSparseFeat(FC.SparseFeat("s_max", 11, 4), maxlen=T, combiner="max")]
        return cols
    return make, x, y


def _model_case(name, *args, **kw):
    """generate_fefm.model_case, then the layer list without the diagonal Embeddings: onn.py declares them but never
    calls them, so they hold no weight (the model_case filter keeps layers that never ran)."""
    GF.model_case(name, *args, **kw)
    path = os.path.join(MODEL_OUT, name + ".npz")
    d = dict(np.load(path))
    meta = json.loads(str(d["meta"]))
    meta["layers"] = [[c, n] for c, n in meta["layers"] if c != "Embedding" or "w_%s/embeddings" % n in d]
    d["meta"] = np.array(json.dumps(meta))
    np.savez_compressed(path, **d)


def fixtures():
    _install()
    GF.MODULES["ONN"] = "deepctr.models.onn"
    GF.MODEL_OUT = MODEL_OUT
    if os.path.isdir(MODEL_OUT):
        shutil.rmtree(MODEL_OUT)
    os.makedirs(MODEL_OUT)

    rng = np.random.RandomState(20261020)
    zero_l2 = dict(l2_reg_linear=0, l2_reg_embedding=0)
    mk, x, y = criteo_like(rng, 32, 6, 3, 4)
    _model_case("onn_defaults", "ONN", GP._columns(mk, dict(zero_l2)), x, y, 81)
    _model_case("onn_reduce_sum", "ONN", GP._columns(mk, dict(reduce_sum=True, dnn_hidden_units=(16, 8), **zero_l2)),
                  x, y, 82)
    _model_case("onn_no_bn", "ONN", GP._columns(mk, dict(use_bn=False, dnn_hidden_units=(16,), **zero_l2)), x, y, 83)
    _model_case("onn_no_dnn", "ONN", GP._columns(mk, dict(dnn_hidden_units=(), **zero_l2)), x, y, 84)
    yr = rng.normal(0, 1, size=32).astype(np.float32)
    _model_case("onn_regression", "ONN", GP._columns(mk, dict(dnn_hidden_units=(16,), task="regression",
                                                                **zero_l2)), x, yr, 85, task="regression")
    mk0, x0, y0 = criteo_like(rng, 32, 5, 0, 8)
    _model_case("onn_no_dense", "ONN", GP._columns(mk0, dict(dnn_hidden_units=(16,), **zero_l2)), x0, y0, 86)
    mk2, x2, y2 = criteo_like(rng, 32, 2, 2, 4)
    _model_case("onn_f2", "ONN", GP._columns(mk2, dict(dnn_hidden_units=(8,), **zero_l2)), x2, y2, 87)
    mkv, xv, yv = _varlen_case(rng)
    _model_case("onn_varlen", "ONN", GP._columns(mkv, dict(dnn_hidden_units=(8,), **zero_l2)), xv, yv, 88)
    mkh, xh, yh = _varlen_case(rng, hashed=True)
    _model_case("onn_hashed", "ONN", GP._columns(mkh, dict(dnn_hidden_units=(8,), reduce_sum=True, **zero_l2)),
                  xh, yh, 89)


def builders():
    import golden_models as G
    import generate_builders as GB
    from golden_models import signature, builder_args
    from deepctr_b200 import backend, engine as E, inputs as I
    from deepctr_b200.layers.normalization import BatchNormalization as BN
    out = {"signatures": {}, "defaults": {}}
    names = sorted(os.path.basename(p)[:-4] for p in os.listdir(MODEL_OUT) if p.endswith(".npz"))
    GB._FILES.update(FILES)
    GP.MODEL_OUT = MODEL_OUT
    with GB._aliased():
        ly = sys.modules["tensorflow.keras.layers"]
        ly.Lambda, ly.Embedding, ly.multiply, ly.BatchNormalization = E.Lambda, I.Embedding, E.multiply, BN
        keras = sys.modules["tensorflow.keras"]
        for name, m in (("backend", backend), ("regularizers", types.SimpleNamespace(l2=E.l2))):
            setattr(keras, name, m)
            sys.modules["tensorflow.keras." + name] = m
        for name in names:
            fx = GP._fixture(name)
            args, kw = builder_args(fx)
            build = GB._reference_builder(os.path.join(REF, "deepctr"), fx.builder)
            E.clear_session()
            model = build(*args, **kw)
            G.weight_map(fx, model)
            out["signatures"][name] = signature(model)
        sig = inspect.signature(GB._reference_builder(os.path.join(REF, "deepctr"), "ONN"))
        out["defaults"]["ONN"] = [[k, repr(p.default)] for k, p in sig.parameters.items()]
        for name in ("backend", "regularizers"):
            sys.modules.pop("tensorflow.keras." + name, None)
    E.clear_session()
    with open(BUILDERS_JSON, "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
    print("wrote", os.path.basename(BUILDERS_JSON), sorted(out["signatures"]))


if __name__ == "__main__":
    fixtures()
    builders()
