#!/usr/bin/env python
"""Generate the FwFM / DeepFEFM fixtures (the builders and their FwFMLayer / FEFMLayer layers) from the REFERENCE's own,
unmodified deepctr/layers/interaction.py, deepctr/models/fwfm.py and deepctr/models/deepfefm.py, executed eagerly
under the torch-backed ``tensorflow`` stand-in of tf_torch_shim.py (the recipe of generate_fibinet.py).

    python tests/golden/generate_fefm.py          (build container only: needs the reference checkout)

Two symbols the two layers and DeepFEFM need are supplied here, so that tf_torch_shim.py and generate_builders.py
(and with them every existing fixture) stay as they are:
  * ``tensorflow.keras.backend.batch_dot`` (the shim exports None), ``tf.scalar_mul`` and ``tf.add_n``, for the
    layers' [B, E] . [B, E] -> [B, 1] products;
  * ``tensorflow.keras.layers.Lambda`` in generate_builders._aliased, for DeepFEFM's ``fefm_logit``.

Keras keeps only the layers reachable from a model's outputs.  The shim's Model lists every layer created, and
DeepFEFM creates a DNN and a Dense(1) that are off the output path when dnn_hidden_units=() (and the linear part
when use_linear=False), so a model fixture records only the weights that receive a gradient and the layers whose
last output is on the loss's autograd graph.

Writes
  tests/golden/fefm/*.npz                   layer level: ``meta``, the input ``x`` [B,F,E], every weight ``w_<name>``,
                                            the output ``out``, an upstream gradient ``dout`` and the gradients
                                            ``gx`` / ``g_<name>``;
  tests/golden/models_fefm/*.npz            model level, the layout of tests/golden/models/;
  tests/golden/reference_builders_fefm.json
                                            the graphs the reference's fwfm.py / deepfefm.py SOURCE FILES build on
                                            this package for those fixtures, and their keyword defaults.
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
import generate_pairwise as GP  # noqa: E402
from generate_models import _collect, _col_meta, keras_loss, kwargs_json, criteo_like  # noqa: E402

REF = "/root/reference"
LAYER_OUT = os.path.join(HERE, "fefm")
MODEL_OUT = os.path.join(HERE, "models_fefm")
BUILDERS_JSON = os.path.join(HERE, "reference_builders_fefm.json")
MODULES = {"FwFM": "deepctr.models.fwfm", "DeepFEFM": "deepctr.models.deepfefm"}
FILES = {"FwFM": ("models/fwfm.py", "models.fwfm"), "DeepFEFM": ("models/deepfefm.py", "models.deepfefm")}


def _batch_dot(x, y, axes=None):
    """tf.keras.backend.batch_dot for the only use here: two [B, E] tensors, axes=1 -> [B, 1]."""
    assert x.dim() == 2 and y.dim() == 2 and axes in (1, [1, 1], (1, 1)), (x.shape, y.shape, axes)
    return (x * y).sum(dim=1, keepdim=True)


def _install():
    S.install(REF)
    tf = sys.modules["tensorflow"]
    tf.scalar_mul = lambda scalar, x, name=None: scalar * x
    tf.add_n = lambda inputs, name=None: sum(inputs[1:], inputs[0])
    sys.modules["tensorflow.keras.backend"].batch_dot = _batch_dot
    importlib.import_module("deepctr.feature_column")
    sys.modules["deepctr.layers.interaction"].batch_dot = _batch_dot     # bound at import time


def layer_case(name, cls, kwargs, B, F, E, seed):
    S.CTX.reset()
    S.CTX.rng = np.random.RandomState(seed)
    S.CTX.grad = True
    L = sys.modules["deepctr.layers.interaction"]
    rng = np.random.RandomState(seed + 1000)
    x = rng.normal(0, 0.5, size=(B, F, E)).astype(np.float32)
    xt = torch.tensor(x, requires_grad=True)
    layer = getattr(L, cls)(**kwargs)
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
    print("%-24s out%s  %d weights" % (name, tuple(d["out"].shape), len(layer._w)))


def _graph_nodes(t):
    seen, stack = set(), [t.grad_fn]
    while stack:
        n = stack.pop()
        if n is None or n in seen:
            continue
        seen.add(n)
        stack.extend(f for f, _ in n.next_functions)
    return seen


def _reachable(layer, nodes):
    outs = [o for o in S._flat(getattr(layer, "_last_out", None)) if isinstance(o, torch.Tensor)]
    with_fn = [o for o in outs if o.grad_fn is not None]
    return not with_fn or any(o.grad_fn in nodes for o in with_fn)


def model_case(name, builder, make_args, x, y, seed, task="binary", note=""):
    """generate_pairwise.model_case, keeping only what is on the output path (see the module docstring)."""
    S.CTX.reset()
    S.CTX.feed = dict(x)
    S.CTX.rng = np.random.RandomState(seed)
    S.CTX.grad = True
    S.CTX.training = None
    FC = sys.modules["deepctr.feature_column"]
    mod = importlib.import_module(MODULES[builder])
    args, kwargs, cols_meta = make_args(FC)
    model = getattr(mod, builder)(*args, **kwargs)
    out = model.outputs
    logit = [l for l in model.layers if l.__class__.__name__ == "PredictionLayer"][-1]._last_in
    loss = keras_loss(task, y, out)
    nodes = _graph_nodes(loss)
    layers = [l for l in model.layers if not l._nested and _reachable(l, nodes)]
    weights = []
    for l in layers:
        weights.extend(_collect(l, l.name + "/"))
    leaves = [t for _, t in weights if t.requires_grad]
    grads = torch.autograd.grad(loss, leaves, allow_unused=True)
    gmap = {id(t): g for t, g in zip(leaves, grads)}
    weights = [(k, t) for k, t in weights if not t.requires_grad or gmap[id(t)] is not None]
    d = {"meta": np.array(json.dumps({"builder": builder, "kwargs": kwargs_json(kwargs), "columns": cols_meta,
                                      "training": None, "task": task, "note": note,
                                      "layers": [[l.__class__.__name__, l.name] for l in layers]}))}
    for k, v in x.items():
        d["x_" + k] = np.asarray(v)
    d["y"] = np.asarray(y, dtype=np.float32)
    for k, t in weights:
        d["w_" + k] = t.detach().numpy().copy()
        if t.requires_grad:
            d["g_" + k] = gmap[id(t)].detach().numpy().copy()
    d["out"] = out.detach().numpy().reshape(-1, 1)
    d["logit"] = logit.detach().numpy().reshape(-1, 1)
    d["loss"] = np.asarray(float(loss.detach()), dtype=np.float64)
    np.savez_compressed(os.path.join(MODEL_OUT, name + ".npz"), **d)
    print("%-28s logit[min %.3f max %.3f] loss %.5f  %d weights" %
          (name, float(d["logit"].min()), float(d["logit"].max()), float(loss.detach()), len(weights)))


def fixtures():
    _install()
    for d in (LAYER_OUT, MODEL_OUT):
        if os.path.isdir(d):
            shutil.rmtree(d)
        os.makedirs(d)

    # ---- layers: FwFMLayer and FEFMLayer at F = 2 (one pair), 7 and 26; E = 4 / 8 -----------------------
    seed = 1
    for cls, tag in (("FwFMLayer", "fwfm"), ("FEFMLayer", "fefm")):
        for F, E_ in ((2, 4), (7, 8), (26, 4)):
            kw = dict(num_fields=F, regularizer=1e-6) if cls == "FwFMLayer" else dict(regularizer=1e-5)
            layer_case("%s_f%d_e%d" % (tag, F, E_), cls, kw, 12, F, E_, seed)
            seed += 1

    rng = np.random.RandomState(20261017)
    zero_l2 = dict(l2_reg_linear=0, l2_reg_embedding=0, l2_reg_field_strength=0)
    # ---- FwFM on a Criteo-like batch with dense features, without a DNN, and over two groups --------------
    mk, x, y = criteo_like(rng, 32, 6, 3, 8)
    model_case("fwfm_criteo", "FwFM", GP._columns(mk, dict(dnn_hidden_units=(16, 8), **zero_l2)), x, y, 41)
    model_case("fwfm_no_dnn", "FwFM", GP._columns(mk, dict(dnn_hidden_units=(), **zero_l2)), x, y, 42)

    n = 32
    xg = {"C%d" % (i + 1): rng.randint(0, 20 + 3 * i, size=n).astype(np.int32) for i in range(7)}
    xg["I1"] = rng.rand(n).astype(np.float32)
    yg = (rng.rand(n) < 0.3).astype(np.float32)

    def group_args(FC):
        cols = [FC.SparseFeat("C%d" % (i + 1), 20 + 3 * i, 4, group_name="g_a" if i < 4 else "g_b")
                for i in range(7)] + [FC.DenseFeat("I1", 1)]
        return (cols, cols), dict(fm_group=("g_a", "g_b"), dnn_hidden_units=(8,), **zero_l2), \
            {"linear": [_col_meta(c, FC) for c in cols], "dnn": [_col_meta(c, FC) for c in cols]}
    model_case("fwfm_two_groups", "FwFM", group_args, xg, yg, 43)

    # ---- DeepFEFM: defaults and each ablation the reference's branches allow ------------------------------
    zero_l2 = dict(l2_reg_linear=0, l2_reg_embedding_feat=0, l2_reg_embedding_field=0)
    mk, x, y = criteo_like(rng, 32, 6, 3, 8)
    for name, kw, sd in (("deepfefm_defaults", {}, 51),
                         ("deepfefm_exclude_feature_embed", dict(exclude_feature_embed_in_dnn=True,
                                                                 dnn_hidden_units=(16, 8)), 52),
                         ("deepfefm_no_fefm_embed_in_dnn", dict(use_fefm_embed_in_dnn=False,
                                                                dnn_hidden_units=(16, 8)), 53),
                         ("deepfefm_linear_fefm", dict(dnn_hidden_units=()), 54),
                         ("deepfefm_no_linear", dict(use_linear=False, dnn_hidden_units=(16, 8)), 55)):
        model_case(name, "DeepFEFM", GP._columns(mk, dict(kw, **zero_l2)), x, y, sd)
    yr = rng.normal(0, 1, size=32).astype(np.float32)
    model_case("deepfefm_regression", "DeepFEFM",
               GP._columns(mk, dict(dnn_hidden_units=(16, 8), task="regression", **zero_l2)), x, yr, 56,
               task="regression")

    # ---- a pooled VarLenSparseFeat among the fields ---------------------------------------------------------
    T = 3
    xv = {"C%d" % (i + 1): rng.randint(0, 20 + 3 * i, size=n).astype(np.int32) for i in range(4)}
    xv["tags"] = rng.randint(0, 15, size=(n, T)).astype(np.int32)
    xv["I1"] = rng.rand(n).astype(np.float32)
    yv = (rng.rand(n) < 0.3).astype(np.float32)

    def varlen_args(FC):
        cols = [FC.SparseFeat("C%d" % (i + 1), 20 + 3 * i, 4) for i in range(4)]
        cols += [FC.VarLenSparseFeat(FC.SparseFeat("tags", 15, 4), maxlen=T, combiner="mean"),
                 FC.DenseFeat("I1", 1)]
        return (cols, cols), dict(dnn_hidden_units=(8,), **zero_l2), \
            {"linear": [_col_meta(c, FC) for c in cols], "dnn": [_col_meta(c, FC) for c in cols]}
    model_case("deepfefm_varlen", "DeepFEFM", varlen_args, xv, yv, 57)


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
        sys.modules["tensorflow.keras.layers"].Lambda = E.Lambda
        for name in names:
            fx = GP._fixture(name)
            args, kw = builder_args(fx)
            build = GB._reference_builder(os.path.join(REF, "deepctr"), fx.builder)
            E.clear_session()
            model = build(*args, **kw)
            G.weight_map(fx, model)
            out["signatures"][name] = signature(model)
        for b in ("FwFM", "DeepFEFM"):
            sig = inspect.signature(GB._reference_builder(os.path.join(REF, "deepctr"), b))
            out["defaults"][b] = [[k, repr(p.default)] for k, p in sig.parameters.items()]
    E.clear_session()
    with open(BUILDERS_JSON, "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
    print("wrote", os.path.basename(BUILDERS_JSON), sorted(out["signatures"]))


if __name__ == "__main__":
    fixtures()
    builders()
