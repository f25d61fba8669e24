#!/usr/bin/env python
"""Generate the EDCN fixtures from the REFERENCE's own, unmodified deepctr/feature_column.py, deepctr/inputs.py,
deepctr/layers/* (RegulationModule in core.py, BridgeModule in interaction.py) and deepctr/models/edcn.py, executed
eagerly under the torch-backed ``tensorflow`` stand-in of tf_torch_shim.py (the recipe of generate_onn.py).

    python tests/golden/generate_edcn.py          (build container only: needs the reference checkout)

The symbols EDCN needs beyond the shim are supplied here, so that tf_torch_shim.py and the other generators (and
with them every existing fixture) stay as they are:
  * ``tensorflow.keras.layers.Reshape`` (edcn.py's Reshape([F, E]) of the bridge output);
  * an ``Activation`` that also knows 'softmax' over the last axis (the output activation of the attention bridge's
    two DNNs), bound where deepctr/layers/activation.py imported the shim's;
  * generate_onn's full Keras BatchNormalization for DNN(use_bn=True), bound where deepctr/layers/core.py imported
    the shim's.  As there, it normalises with the batch statistics and stores them as the moving statistics, so a
    prediction and a training step compare against the same recorded outputs.  The reference's DNN keeps these
    layers in ``bn_layers``; the fixture keys name them ``bn<i>``, as the package's DNN does.
For the graphs built from the reference's edcn.py on this package, generate_builders._aliased is given the package's
Reshape.

Writes
  tests/golden/models_edcn/*.npz             model level, the layout of tests/golden/models/;
  tests/golden/reference_builders_edcn.json  the graphs the reference's edcn.py SOURCE FILE builds on this package for
                                             those fixtures, and its keyword defaults.
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
import generate_onn as GO  # noqa: E402
import generate_pairwise as GP  # noqa: E402
from generate_models import criteo_like  # noqa: E402

REF = GF.REF
MODEL_OUT = os.path.join(HERE, "models_edcn")
BUILDERS_JSON = os.path.join(HERE, "reference_builders_edcn.json")
FILES = {"EDCN": ("models/edcn.py", "models.edcn")}


class Reshape(S.Layer):
    """tf.keras.layers.Reshape(target_shape): the per-sample shape becomes ``target_shape``."""

    def __init__(self, target_shape, **kw):
        S.Layer.__init__(self, **kw)
        self.target_shape = tuple(int(s) for s in target_shape)

    def call(self, x, **kw):
        return x.reshape((x.shape[0],) + self.target_shape)


class Activation(S.Activation):
    """The shim's Activation plus 'softmax' over the last axis (tf.keras.activations.softmax)."""

    def call(self, x, **kwargs):
        if self.activation == "softmax":
            return torch.softmax(x, dim=-1)
        return S.Activation.call(self, x)


def _install():
    S.install(REF)
    sys.modules["tensorflow.keras.layers"].Reshape = Reshape
    importlib.import_module("deepctr.feature_column")
    sys.modules["deepctr.layers.activation"].Activation = Activation
    sys.modules["deepctr.layers.core"].BatchNormalization = GO.BatchNormalization


def _model_case(name, *args, **kw):
    """generate_fefm.model_case, then the DNN's ``bn_layers<i>`` keys renamed ``bn<i>``."""
    GF.model_case(name, *args, **kw)
    path = os.path.join(MODEL_OUT, name + ".npz")
    d = dict(np.load(path))
    d = {k.replace("/bn_layers", "/bn"): v for k, v in d.items()}
    np.savez_compressed(path, **d)


def _varlen_case(rng, n=32, T=4):
    """Two single-valued fields and a mean-pooled varlen field (padding id 0 masked), E = 4."""
    lens = rng.randint(1, T + 1, size=n).astype(np.int32)
    seq = rng.randint(1, 13, size=(n, T)).astype(np.int32)
    seq[np.arange(T)[None, :] >= lens[:, None]] = 0
    x = {"C1": rng.randint(0, 20, size=n).astype(np.int32), "C2": rng.randint(0, 23, size=n).astype(np.int32),
         "S1": seq}
    y = (rng.rand(n) < 0.3).astype(np.float32)

    def make(FC):
        return [FC.SparseFeat("C1", 20, 4), FC.SparseFeat("C2", 23, 4),
                FC.VarLenSparseFeat(FC.SparseFeat("S1", 13, 4), maxlen=T, combiner="mean")]
    return make, x, y


def fixtures():
    _install()
    GF.MODULES["EDCN"] = "deepctr.models.edcn"
    GF.MODEL_OUT = MODEL_OUT
    if os.path.isdir(MODEL_OUT):
        shutil.rmtree(MODEL_OUT)
    os.makedirs(MODEL_OUT)

    rng = np.random.RandomState(20261021)
    zero_l2 = dict(l2_reg_linear=0, l2_reg_embedding=0, l2_reg_cross=0)
    # ---- the reference test's four configurations (tests/models/EDCN_test.py) ---------------------------------
    seed = 91
    for bridge, cross_num, param, F in (("pointwise_addition", 2, "vector", 3), ("hadamard_product", 2, "vector", 4),
                                        ("concatenation", 1, "vector", 5), ("attention_pooling", 2, "matrix", 6)):
        mk, x, y = criteo_like(rng, 32, F, 0, 4)
        kw = dict(cross_num=cross_num, cross_parameterization=param, bridge_type=bridge, **zero_l2)
        _model_case("edcn_%s" % bridge, "EDCN", GP._columns(mk, kw), x, y, seed)
        seed += 1
    # ---- the defaults on 26 Criteo-like fields ------------------------------------------------------------------
    mk, x, y = criteo_like(rng, 32, 26, 0, 4)
    _model_case("edcn_defaults", "EDCN", GP._columns(mk, dict(zero_l2)), x, y, 95)
    # ---- tau = 0.5 over three layers, BatchNormalization in the DNNs, a pooled field, regression ----------------
    mk, x, y = criteo_like(rng, 32, 5, 0, 4)
    _model_case("edcn_tau_half", "EDCN", GP._columns(mk, dict(tau=0.5, cross_num=3, bridge_type="hadamard_product",
                                                               **zero_l2)), x, y, 96)
    _model_case("edcn_dnn_bn", "EDCN", GP._columns(mk, dict(dnn_use_bn=True, bridge_type="attention_pooling",
                                                             **zero_l2)), x, y, 97)
    mkv, xv, yv = _varlen_case(rng)
    _model_case("edcn_varlen", "EDCN", GP._columns(mkv, dict(bridge_type="pointwise_addition", **zero_l2)),
                xv, yv, 98)
    yr = rng.normal(0, 1, size=32).astype(np.float32)
    _model_case("edcn_regression", "EDCN", GP._columns(mk, dict(task="regression", **zero_l2)), x, yr, 99,
                task="regression")


def builders():
    import golden_models as G
    import generate_builders as GB
    from golden_models import signature, builder_args
    from deepctr_b200 import engine as E
    out = {"signatures": {}, "defaults": {}}
    names = sorted(os.path.basename(p)[:-4] for p in os.listdir(MODEL_OUT) if p.endswith(".npz"))
    GB._FILES.update(FILES)
    GP.MODEL_OUT = MODEL_OUT
    with GB._aliased():
        sys.modules["tensorflow.keras.layers"].Reshape = E.Reshape
        for name in names:
            fx = GP._fixture(name)
            args, kw = builder_args(fx)
            build = GB._reference_builder(os.path.join(REF, "deepctr"), fx.builder)
            E.clear_session()
            model = build(*args, **kw)
            G.weight_map(fx, model)
            out["signatures"][name] = signature(model)
        sig = inspect.signature(GB._reference_builder(os.path.join(REF, "deepctr"), "EDCN"))
        out["defaults"]["EDCN"] = [[k, repr(p.default)] for k, p in sig.parameters.items()]
    E.clear_session()
    with open(BUILDERS_JSON, "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
    print("wrote", os.path.basename(BUILDERS_JSON), sorted(out["signatures"]))


if __name__ == "__main__":
    fixtures()
    builders()
