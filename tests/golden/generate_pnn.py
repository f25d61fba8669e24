#!/usr/bin/env python
"""Generate the PNN fixtures (the builder and its InnerProductLayer / OutterProductLayer layers) from the REFERENCE's
own, unmodified deepctr/layers/interaction.py and deepctr/models/pnn.py, executed eagerly under the torch-backed
``tensorflow`` stand-in of tf_torch_shim.py (the recipe of generate_fefm.py).

    python tests/golden/generate_pnn.py          (build container only: needs the reference checkout)

One symbol PNN needs is supplied here, so that tf_torch_shim.py and generate_builders.py (and with them every
existing fixture) stay as they are: ``tensorflow.keras.layers.Reshape``, for the shim (a per-sample reshape) and in
generate_builders._aliased (deepctr_b200.engine.Reshape).

PNN always creates and calls both product layers; the one a model does not use is off the output path, so a model
fixture records only the weights that receive a gradient and the layers on the loss's autograd graph
(generate_fefm.model_case).  Dropout stays 0: Keras' dropout RNG is not pinned.

Writes
  tests/golden/pnn/*.npz                    layer level: ``meta``, the input ``x`` [B,F,E] (the layer is called on
                                            its F [B,1,E] slices), the weight ``w_kernel``, the output ``out``, an
                                            upstream gradient ``dout`` and the gradients ``gx`` / ``g_kernel``;
  tests/golden/models_pnn/*.npz             model level, the layout of tests/golden/models/;
  tests/golden/reference_builders_pnn.json  the graphs the reference's pnn.py SOURCE FILE builds on this package for
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
import generate_pairwise as GP  # noqa: E402
from generate_models import _col_meta, criteo_like  # noqa: E402

REF = GF.REF
LAYER_OUT = os.path.join(HERE, "pnn")
MODEL_OUT = os.path.join(HERE, "models_pnn")
BUILDERS_JSON = os.path.join(HERE, "reference_builders_pnn.json")
FILES = {"PNN": ("models/pnn.py", "models.pnn")}


class Reshape(S.Layer):
    """keras.layers.Reshape(target_shape) on the shim: the per-sample shape becomes target_shape."""

    def __init__(self, target_shape, **kwargs):
        S.Layer.__init__(self, **kwargs)
        self.target_shape = tuple(int(s) for s in target_shape)

    def call(self, x, **kw):
        return x.reshape((x.shape[0],) + self.target_shape)


def _install():
    S.install(REF)
    sys.modules["tensorflow.keras.layers"].Reshape = Reshape
    importlib.import_module("deepctr.feature_column")


def layer_case(name, cls, kwargs, B, F, E, seed):
    S.CTX.reset()
    S.CTX.rng = np.random.RandomState(seed)
    S.CTX.grad = True
    L = sys.modules["deepctr.layers.interaction"]
    rng = np.random.RandomState(seed + 1000)
    x = rng.normal(0, 0.5, size=(B, F, E)).astype(np.float32)
    xt = torch.tensor(x, requires_grad=True)
    layer = getattr(L, cls)(**kwargs)
    out = layer(list(torch.split(xt, 1, dim=1)))
    dout = rng.normal(0, 1.0, size=tuple(out.shape)).astype(np.float32)
    leaves = [t for _, t in layer._w]
    grads = torch.autograd.grad((out * torch.as_tensor(dout)).sum(), [xt] + leaves)
    d = {"meta": np.array(json.dumps({"layer": cls, "kwargs": kwargs})), "x": x,
         "out": out.detach().numpy(), "dout": dout, "gx": grads[0].numpy()}
    for (wn, t), g in zip(layer._w, grads[1:]):
        d["w_" + wn] = t.detach().numpy().copy()
        d["g_" + wn] = g.numpy()
    np.savez_compressed(os.path.join(LAYER_OUT, name + ".npz"), **d)
    print("%-24s out%s  %d weights" % (name, tuple(d["out"].shape), len(layer._w)))


def _pnn_columns(mk, extra_kw):
    """PNN takes the DNN columns only (pnn.py:18): the fixture records them under 'dnn' and no linear columns."""
    def f(FC):
        cols = mk(FC)
        return (cols,), dict(extra_kw), {"linear": [], "dnn": [_col_meta(c, FC) for c in cols]}
    return f


def fixtures():
    _install()
    GF.MODULES["PNN"] = "deepctr.models.pnn"
    GF.MODEL_OUT = MODEL_OUT
    for d in (LAYER_OUT, MODEL_OUT):
        if os.path.isdir(d):
            shutil.rmtree(d)
        os.makedirs(d)

    # ---- layers: inner (reduce_sum True / False) and outer (mat / vec / num) at F = 2, 7, 26; E = 4 / 8 -------
    seed = 1
    for tag, cls, kw in (("inner", "InnerProductLayer", {}),
                         ("inner_elementwise", "InnerProductLayer", dict(reduce_sum=False)),
                         ("outer_mat", "OutterProductLayer", dict(kernel_type="mat", seed=1024)),
                         ("outer_vec", "OutterProductLayer", dict(kernel_type="vec", seed=1024)),
                         ("outer_num", "OutterProductLayer", dict(kernel_type="num", seed=1024))):
        for F, E_ in ((2, 4), (7, 8), (26, 4)):
            layer_case("%s_f%d_e%d" % (tag, F, E_), cls, kw, 12, F, E_, seed)
            seed += 1

    rng = np.random.RandomState(20261018)
    zero_l2 = dict(l2_reg_embedding=0)
    small = dict(dnn_hidden_units=(16, 8), **zero_l2)
    mk, x, y = criteo_like(rng, 32, 6, 3, 8)
    for name, kw, sd in (("pnn_defaults", dict(zero_l2), 61),
                         ("pnn_opnn_mat", dict(use_inner=False, use_outter=True, **small), 62),
                         ("pnn_opnn_vec", dict(use_inner=False, use_outter=True, kernel_type="vec", **small), 63),
                         ("pnn_opnn_num", dict(use_inner=False, use_outter=True, kernel_type="num", **small), 64),
                         ("pnn_inner_outer_mat", dict(use_outter=True, **small), 65),
                         ("pnn_no_products", dict(use_inner=False, **small), 66)):
        GF.model_case(name, "PNN", _pnn_columns(mk, kw), x, y, sd)
    yr = rng.normal(0, 1, size=32).astype(np.float32)
    GF.model_case("pnn_regression", "PNN", _pnn_columns(mk, dict(task="regression", **small)), x, yr, 67,
                  task="regression")

    mk_nd, x_nd, y_nd = criteo_like(rng, 32, 5, 0, 4)
    GF.model_case("pnn_no_dense", "PNN", _pnn_columns(mk_nd, dict(use_outter=True, **small)), x_nd, y_nd, 68)

    # ---- a pooled VarLenSparseFeat among the fields ---------------------------------------------------------
    n, T = 32, 3
    xv = {"C%d" % (i + 1): rng.randint(0, 20 + 3 * i, size=n).astype(np.int32) for i in range(4)}
    xv["tags"] = rng.randint(0, 15, size=(n, T)).astype(np.int32)
    xv["I1"] = rng.rand(n).astype(np.float32)
    yv = (rng.rand(n) < 0.3).astype(np.float32)

    def varlen_cols(FC):
        cols = [FC.SparseFeat("C%d" % (i + 1), 20 + 3 * i, 4) for i in range(4)]
        return cols + [FC.VarLenSparseFeat(FC.SparseFeat("tags", 15, 4), maxlen=T, combiner="mean"),
                       FC.DenseFeat("I1", 1)]
    GF.model_case("pnn_varlen", "PNN", _pnn_columns(varlen_cols, dict(use_outter=True, kernel_type="vec",
                                                                      dnn_hidden_units=(8,), **zero_l2)),
                  xv, yv, 69)


def builders():
    import golden_models as G
    import generate_builders as GB
    from test_reference_builders_dropin import signature
    from test_pnn_goldens import pnn_builder_args
    from deepctr_b200 import engine as E
    out = {"signatures": {}, "defaults": {}}
    names = sorted(os.path.basename(p)[:-4] for p in os.listdir(MODEL_OUT) if p.endswith(".npz"))
    GB._FILES.update(FILES)
    GP.MODEL_OUT = MODEL_OUT
    with GB._aliased():
        sys.modules["tensorflow.keras.layers"].Reshape = E.Reshape
        for name in names:
            fx = GP._fixture(name)
            args, kw = pnn_builder_args(fx)
            build = GB._reference_builder(os.path.join(REF, "deepctr"), fx.builder)
            E.clear_session()
            model = build(*args, **kw)
            G.weight_map(fx, model)
            out["signatures"][name] = signature(model)
        sig = inspect.signature(GB._reference_builder(os.path.join(REF, "deepctr"), "PNN"))
        out["defaults"]["PNN"] = [[k, repr(p.default)] for k, p in sig.parameters.items()]
    E.clear_session()
    with open(BUILDERS_JSON, "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
    print("wrote", os.path.basename(BUILDERS_JSON), sorted(out["signatures"]))


if __name__ == "__main__":
    fixtures()
    builders()
