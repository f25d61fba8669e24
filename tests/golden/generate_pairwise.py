#!/usr/bin/env python
"""Generate the pairwise-interaction fixtures (NFM / AFM and their layers) from the REFERENCE's own, unmodified
deepctr/layers/interaction.py (AFMLayer, BiInteractionPooling), deepctr/models/nfm.py and deepctr/models/afm.py,
executed eagerly under the torch-backed ``tensorflow`` stand-in of tf_torch_shim.py.

    python tests/golden/generate_pairwise.py          (build container only: needs /root/reference)

Writes
  tests/golden/pairwise/*.npz               layer level: ``meta``, the input ``x`` [B,F,E], every weight ``w_<name>``,
                                            the output ``out``, an upstream gradient ``dout`` and the gradients
                                            ``gx`` / ``g_<name>`` of <out, dout> by torch autograd through the layer;
  tests/golden/models_pairwise/*.npz        model level, the layout of tests/golden/models/ (generate_models.py);
  tests/golden/reference_builders_pairwise.json
                                            the graphs the reference's nfm.py / afm.py SOURCE FILES build on this
                                            package for those fixtures, and their keyword defaults (the layout of
                                            reference_builders.json, generate_builders.py).
The existing fixture directories and reference_builders.json are not touched.
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
from generate_models import _collect, _col_meta, keras_loss, kwargs_json, criteo_like  # noqa: E402

REF = "/root/reference"
LAYER_OUT = os.path.join(HERE, "pairwise")
MODEL_OUT = os.path.join(HERE, "models_pairwise")
BUILDERS_JSON = os.path.join(HERE, "reference_builders_pairwise.json")
MODULES = {"NFM": "deepctr.models.nfm", "AFM": "deepctr.models.afm"}
FILES = {"NFM": "models/nfm.py", "AFM": "models/afm.py"}


# ---- layer level ----------------------------------------------------------------------------------
def layer_case(name, cls, kwargs, B, F, E, seed):
    S.CTX.reset()
    S.CTX.rng = np.random.RandomState(seed)
    S.CTX.grad = True
    L = sys.modules["deepctr.layers.interaction"]
    rng = np.random.RandomState(seed + 1000)
    x = rng.normal(0, 0.5, size=(B, F, E)).astype(np.float32)
    xt = torch.tensor(x, requires_grad=True)
    layer = getattr(L, cls)(**kwargs)
    if cls == "AFMLayer":
        out = layer(list(torch.split(xt, 1, dim=1)))
    else:
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
    print("%-28s out%s" % (name, tuple(d["out"].shape)))


# ---- model level (generate_models.run_case for the NFM / AFM builder modules) -------------------
def model_case(name, builder, make_args, x, y, seed, task="binary", note=""):
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
    weights = []
    for l in model.layers:
        if not l._nested:
            weights.extend(_collect(l, l.name + "/"))
    leaves = [t for _, t in weights if t.requires_grad]
    grads = torch.autograd.grad(loss, leaves, allow_unused=True)
    gmap = {id(t): g for t, g in zip(leaves, grads)}
    d = {"meta": np.array(json.dumps({"builder": builder, "kwargs": kwargs_json(kwargs), "columns": cols_meta,
                                      "training": None, "task": task, "note": note,
                                      "layers": [[l.__class__.__name__, l.name] for l in model.layers
                                                 if not l._nested]}))}
    for k, v in x.items():
        d["x_" + k] = np.asarray(v)
    d["y"] = np.asarray(y, dtype=np.float32)
    for k, t in weights:
        d["w_" + k] = t.detach().numpy().copy()
        if t.requires_grad:
            g = gmap.get(id(t))
            d["g_" + k] = (g if g is not None else torch.zeros_like(t)).detach().numpy().copy()
    d["out"] = out.detach().numpy().reshape(-1, 1)
    d["logit"] = logit.detach().numpy().reshape(-1, 1)
    d["loss"] = np.asarray(float(loss.detach()), dtype=np.float64)
    np.savez_compressed(os.path.join(MODEL_OUT, name + ".npz"), **d)
    print("%-28s logit[min %.3f max %.3f] loss %.5f  %d weights" %
          (name, float(d["logit"].min()), float(d["logit"].max()), float(loss.detach()), len(weights)))


def _columns(mk, extra_kw):
    def f(FC):
        cols = mk(FC)
        return (cols, cols), dict(extra_kw), \
            {"linear": [_col_meta(c, FC) for c in cols], "dnn": [_col_meta(c, FC) for c in cols]}
    return f


def fixtures():
    S.install(REF)
    importlib.import_module("deepctr.feature_column")
    for d in (LAYER_OUT, MODEL_OUT):
        if os.path.isdir(d):
            shutil.rmtree(d)
        os.makedirs(d)

    # ---- layers: AFMLayer at P = 1 (F = 2), F = 7 and F = 26; E 4 / 8, A 1 / 4; BiInteractionPooling
    layer_case("afm_f2_e4_a1", "AFMLayer", dict(attention_factor=1), 16, 2, 4, 1)
    layer_case("afm_f7_e8_a4", "AFMLayer", dict(attention_factor=4), 16, 7, 8, 2)
    layer_case("afm_f26_e4_a4", "AFMLayer", dict(attention_factor=4), 12, 26, 4, 3)
    layer_case("afm_f26_e8_a1", "AFMLayer", dict(attention_factor=1, l2_reg_w=0.01), 12, 26, 8, 4)
    layer_case("bi_interaction_f7_e8", "BiInteractionPooling", {}, 16, 7, 8, 5)
    layer_case("bi_interaction_f26_e4", "BiInteractionPooling", {}, 12, 26, 4, 6)

    rng = np.random.RandomState(20261015)
    # ---- NFM on a Criteo-like batch with dense features (examples/run_classification_criteo.py shape) ----
    mk, x, y = criteo_like(rng, 32, 6, 3, 8)
    model_case("nfm_criteo", "NFM", _columns(mk, dict(dnn_hidden_units=(16, 8), l2_reg_linear=0,
                                                       l2_reg_embedding=0)), x, y, 21)
    model_case("nfm_no_dnn", "NFM", _columns(mk, dict(dnn_hidden_units=(), l2_reg_linear=0, l2_reg_embedding=0)),
               x, y, 22)

    # ---- AFM: no DenseFeat (support_dense=False); attention over two groups, and the FM variant -------
    n = 32
    xa = {"C%d" % (i + 1): rng.randint(0, 20 + 3 * i, size=n).astype(np.int32) for i in range(7)}
    ya = (rng.rand(n) < 0.3).astype(np.float32)

    def afm_cols(FC):
        return [FC.SparseFeat("C%d" % (i + 1), 20 + 3 * i, 8, group_name="g_a" if i < 4 else "g_b")
                for i in range(7)]

    def afm_args(kw):
        def f(FC):
            cols = afm_cols(FC)
            return (cols, cols), dict(kw), \
                {"linear": [_col_meta(c, FC) for c in cols], "dnn": [_col_meta(c, FC) for c in cols]}
        return f
    model_case("afm_two_groups", "AFM", afm_args(dict(fm_group=("g_a", "g_b"), attention_factor=4,
                                                     l2_reg_linear=0, l2_reg_embedding=0, l2_reg_att=0)),
               xa, ya, 23)
    mk4, x4, y4 = criteo_like(rng, 32, 6, 0, 4)
    model_case("afm_fm_only", "AFM", _columns(mk4, dict(use_attention=False, l2_reg_linear=0, l2_reg_embedding=0)),
               x4, y4, 24)


# ---- builder graphs: the reference's builder sources executed on this package -----------------------
def builders():
    import golden_models as G
    import generate_builders as GB
    from golden_models import signature, builder_args
    from deepctr_b200 import engine as E
    from deepctr_b200.layers.normalization import Dropout
    out = {"signatures": {}, "defaults": {}}
    names = sorted(os.path.basename(p)[:-4] for p in os.listdir(MODEL_OUT) if p.endswith(".npz"))
    GB._FILES.update({"NFM": (FILES["NFM"], "models.nfm"), "AFM": (FILES["AFM"], "models.afm")})
    with GB._aliased():
        sys.modules["tensorflow.keras.layers"].Dropout = Dropout
        for name in names:
            fx = _fixture(name)
            args, kw = builder_args(fx)
            build = GB._reference_builder(os.path.join(REF, "deepctr"), fx.builder)
            E.clear_session()
            model = build(*args, **kw)
            G.weight_map(fx, model)
            out["signatures"][name] = signature(model)
        for b in ("NFM", "AFM"):
            sig = inspect.signature(GB._reference_builder(os.path.join(REF, "deepctr"), b))
            out["defaults"][b] = [[k, repr(p.default)] for k, p in sig.parameters.items()]
    E.clear_session()
    with open(BUILDERS_JSON, "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
    print("wrote", os.path.basename(BUILDERS_JSON), sorted(out["signatures"]))


def _fixture(name):
    import golden_models as G
    fx = G.Fixture.__new__(G.Fixture)
    d = np.load(os.path.join(MODEL_OUT, name + ".npz"))
    fx.name = name
    fx.meta = json.loads(str(d["meta"]))
    fx.x = {k[2:]: d[k] for k in d.files if k.startswith("x_")}
    fx.y = d["y"]
    fx.w = {k[2:]: d[k] for k in d.files if k.startswith("w_")}
    fx.g = {k[2:]: d[k] for k in d.files if k.startswith("g_")}
    fx.out, fx.logit, fx.loss = d["out"], d["logit"], float(d["loss"])
    fx.builder, fx.kwargs = fx.meta["builder"], fx.meta["kwargs"]
    fx.task = fx.meta.get("task", "binary")
    fx.training = bool(fx.meta.get("training"))
    return fx


if __name__ == "__main__":
    fixtures()
    builders()
