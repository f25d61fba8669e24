#!/usr/bin/env python
"""Generate the FiBiNET fixtures (the builder and its SENETLayer / BilinearInteraction layers) from the REFERENCE's own,
unmodified deepctr/layers/interaction.py and deepctr/models/fibinet.py, executed eagerly under the torch-backed
``tensorflow`` stand-in of tf_torch_shim.py (the recipe of generate_pairwise.py).

    python tests/golden/generate_fibinet.py          (build container only: needs the reference checkout)

Writes
  tests/golden/fibinet/*.npz                layer level: ``meta``, the input ``x`` [B,F,E], every weight ``w_<name>``,
                                            the output ``out`` (SENET: its F outputs concatenated on axis 1), an
                                            upstream gradient ``dout`` and the gradients ``gx`` / ``g_<name>``;
  tests/golden/models_fibinet/*.npz         model level, the layout of tests/golden/models/;
  tests/golden/reference_builders_fibinet.json
                                            the graphs the reference's fibinet.py SOURCE FILE builds on this package
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
import generate_pairwise as GP  # noqa: E402
from generate_models import _col_meta, criteo_like  # noqa: E402

REF = "/root/reference"
LAYER_OUT = os.path.join(HERE, "fibinet")
MODEL_OUT = os.path.join(HERE, "models_fibinet")
BUILDERS_JSON = os.path.join(HERE, "reference_builders_fibinet.json")


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
    if isinstance(out, (list, tuple)):
        out = torch.cat(list(out), dim=1)
    dout = rng.normal(0, 1.0, size=tuple(out.shape)).astype(np.float32)
    leaves = [t for _, t in layer._w]
    grads = torch.autograd.grad((out * torch.as_tensor(dout)).sum(), [xt] + leaves)
    d = {"meta": np.array(json.dumps({"layer": cls, "kwargs": kwargs})), "x": x,
         "out": out.detach().numpy(), "dout": dout, "gx": grads[0].numpy()}
    for (wn, t), g in zip(layer._w, grads[1:]):
        d["w_" + wn] = t.detach().numpy().copy()
        d["g_" + wn] = g.numpy()
    np.savez_compressed(os.path.join(LAYER_OUT, name + ".npz"), **d)
    print("%-32s out%s  %d weights" % (name, tuple(d["out"].shape), len(layer._w)))


def fixtures():
    S.install(REF)
    importlib.import_module("deepctr.feature_column")
    for d in (LAYER_OUT, MODEL_OUT):
        if os.path.isdir(d):
            shutil.rmtree(d)
        os.makedirs(d)
    GP.MODEL_OUT = MODEL_OUT
    GP.MODULES["FiBiNET"] = "deepctr.models.fibinet"

    # ---- layers: SENET at F = 2 with ratio 3 (reduction size max(1, 0) = 1), F = 7 and 26 -------------
    layer_case("senet_f2_r3_e4", "SENETLayer", dict(reduction_ratio=3), 16, 2, 4, 1)
    layer_case("senet_f7_r2_e8", "SENETLayer", dict(reduction_ratio=2), 16, 7, 8, 2)
    layer_case("senet_f26_r3_e4", "SENETLayer", dict(reduction_ratio=3), 12, 26, 4, 3)
    # ---- BilinearInteraction x {all, each, interaction} at F = 2, 7, 26 and E = 4, 8 --------------------
    seed = 10
    for t in ("all", "each", "interaction"):
        for F, E_ in ((2, 4), (7, 8), (26, 4)):
            layer_case("bilinear_%s_f%d_e%d" % (t, F, E_), "BilinearInteraction", dict(bilinear_type=t), 12, F, E_,
                       seed)
            seed += 1

    rng = np.random.RandomState(20261016)
    # ---- FiBiNET on a Criteo-like batch with dense features, each bilinear type, and no DNN -------------
    mk, x, y = criteo_like(rng, 32, 6, 3, 8)
    for t, hu, sd in (("interaction", (16, 8), 31), ("all", (16, 8), 32), ("each", (16, 8), 33),
                      ("interaction", (), 34)):
        name = "fibinet_%s" % t if hu else "fibinet_no_dnn"
        GP.model_case(name, "FiBiNET", GP._columns(mk, dict(bilinear_type=t, dnn_hidden_units=hu, l2_reg_linear=0,
                                                            l2_reg_embedding=0)), x, y, sd)

    # ---- a pooled VarLenSparseFeat among the fields -----------------------------------------------------
    n, T = 32, 3
    xv = {"C%d" % (i + 1): rng.randint(0, 20 + 3 * i, size=n).astype(np.int32) for i in range(4)}
    xv["tags"] = rng.randint(0, 15, size=(n, T)).astype(np.int32)
    xv["I1"] = rng.rand(n).astype(np.float32)
    yv = (rng.rand(n) < 0.3).astype(np.float32)

    def varlen_args(FC):
        cols = [FC.SparseFeat("C%d" % (i + 1), 20 + 3 * i, 4) for i in range(4)]
        cols += [FC.VarLenSparseFeat(FC.SparseFeat("tags", 15, 4), maxlen=T, combiner="mean"),
                 FC.DenseFeat("I1", 1)]
        return (cols, cols), dict(bilinear_type="each", reduction_ratio=2, dnn_hidden_units=(8,), l2_reg_linear=0,
                                  l2_reg_embedding=0), \
            {"linear": [_col_meta(c, FC) for c in cols], "dnn": [_col_meta(c, FC) for c in cols]}
    GP.model_case("fibinet_varlen", "FiBiNET", varlen_args, xv, yv, 35)


def builders():
    import golden_models as G
    import generate_builders as GB
    from golden_models import signature, builder_args
    from deepctr_b200 import engine as E
    out = {"signatures": {}, "defaults": {}}
    names = sorted(os.path.basename(p)[:-4] for p in os.listdir(MODEL_OUT) if p.endswith(".npz"))
    GB._FILES["FiBiNET"] = ("models/fibinet.py", "models.fibinet")
    GP.MODEL_OUT = MODEL_OUT
    with GB._aliased():
        for name in names:
            fx = GP._fixture(name)
            args, kw = builder_args(fx)
            build = GB._reference_builder(os.path.join(REF, "deepctr"), fx.builder)
            E.clear_session()
            model = build(*args, **kw)
            G.weight_map(fx, model)
            out["signatures"][name] = signature(model)
        sig = inspect.signature(GB._reference_builder(os.path.join(REF, "deepctr"), "FiBiNET"))
        out["defaults"]["FiBiNET"] = [[k, repr(p.default)] for k, p in sig.parameters.items()]
    E.clear_session()
    with open(BUILDERS_JSON, "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
    print("wrote", os.path.basename(BUILDERS_JSON), sorted(out["signatures"]))


if __name__ == "__main__":
    fixtures()
    builders()
