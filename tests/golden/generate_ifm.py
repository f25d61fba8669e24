#!/usr/bin/env python
"""Generate the IFM / DIFM fixtures from the REFERENCE's own, unmodified deepctr/feature_column.py (the refined linear
term of get_linear_logit), deepctr/models/ifm.py and deepctr/models/difm.py, executed eagerly under the torch-backed
``tensorflow`` stand-in of tf_torch_shim.py (the recipe of generate_pnn.py).

    python tests/golden/generate_ifm.py          (build container only: needs the reference checkout)

One symbol IFM needs is supplied here, so that tf_torch_shim.py and generate_builders.py (and with them every existing
fixture) stay as they are: ``tf.shape`` (a 1-D integer tensor, so that IFM's ``tf.cast(tf.shape(x)[-1], tf.float32)``
is the field count as a float), and ``tensorflow.keras.layers.Lambda`` in generate_builders._aliased.  Dropout stays
0: Keras' dropout RNG is not pinned.

Writes
  tests/golden/models_ifm/*.npz             model level, the layout of tests/golden/models/;
  tests/golden/reference_builders_ifm.json  the graphs the reference's ifm.py / difm.py SOURCE FILES build on this
                                            package for those fixtures, and their keyword defaults.
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
MODEL_OUT = os.path.join(HERE, "models_ifm")
BUILDERS_JSON = os.path.join(HERE, "reference_builders_ifm.json")
MODULES = {"IFM": "deepctr.models.ifm", "DIFM": "deepctr.models.difm"}
FILES = {"IFM": ("models/ifm.py", "models.ifm"), "DIFM": ("models/difm.py", "models.difm")}


def _install():
    S.install(REF)
    sys.modules["tensorflow"].shape = lambda x, **kw: torch.tensor(list(x.shape))
    importlib.import_module("deepctr.feature_column")


def _varlen_case(rng, n=32, T=4):
    """The columns of the reference's tests/utils.py get_test_data: single-valued sparse features, a dense feature,
    pooled varlen features with the combiners sum / mean / max, and a weighted sequence with a length input.  Every
    categorical column is a field of F."""
    lens = rng.randint(1, T + 1, size=n).astype(np.int32)

    def padded(vocab):
        a = rng.randint(1, vocab, size=(n, T)).astype(np.int32)
        a[np.arange(T)[None, :] >= lens[:, None]] = 0
        return a
    x = {"C1": rng.randint(0, 20, size=n).astype(np.int32), "C2": rng.randint(0, 23, size=n).astype(np.int32),
         "C3": rng.randint(0, 26, size=n).astype(np.int32), "I1": rng.rand(n).astype(np.float32),
         "s_sum": padded(13), "s_mean": padded(15), "s_max": padded(11), "s_w": padded(17),
         "s_w_len": lens.copy(), "s_w_weight": rng.rand(n, T, 1).astype(np.float32)}
    y = (rng.rand(n) < 0.3).astype(np.float32)

    def make(FC):
        cols = [FC.SparseFeat("C1", 20, 4), FC.SparseFeat("C2", 23, 4), FC.SparseFeat("C3", 26, 4),
                FC.DenseFeat("I1", 1)]
        cols += [FC.VarLenSparseFeat(FC.SparseFeat("s_sum", 13, 4), maxlen=T, combiner="sum"),
                 FC.VarLenSparseFeat(FC.SparseFeat("s_mean", 15, 4), maxlen=T, combiner="mean"),
                 FC.VarLenSparseFeat(FC.SparseFeat("s_max", 11, 4), maxlen=T, combiner="max"),
                 FC.VarLenSparseFeat(FC.SparseFeat("s_w", 17, 4), maxlen=T, combiner="sum", length_name="s_w_len",
                                     weight_name="s_w_weight", weight_norm=True)]
        return cols
    return make, x, y


def fixtures():
    _install()
    GF.MODULES.update(MODULES)
    GF.MODEL_OUT = MODEL_OUT
    if os.path.isdir(MODEL_OUT):
        shutil.rmtree(MODEL_OUT)
    os.makedirs(MODEL_OUT)

    rng = np.random.RandomState(20261019)
    zero_l2 = dict(l2_reg_linear=0, l2_reg_embedding=0)
    mk, x, y = criteo_like(rng, 32, 6, 3, 8)
    GF.model_case("ifm_criteo", "IFM", GP._columns(mk, dict(dnn_hidden_units=(16, 8), **zero_l2)), x, y, 71)
    yr = rng.normal(0, 1, size=32).astype(np.float32)
    GF.model_case("ifm_regression", "IFM", GP._columns(mk, dict(dnn_hidden_units=(16,), task="regression",
                                                                **zero_l2)), x, yr, 72, task="regression")
    GF.model_case("difm_defaults", "DIFM", GP._columns(mk, dict(zero_l2)), x, y, 73)
    GF.model_case("difm_no_att_res", "DIFM", GP._columns(mk, dict(att_res=False, dnn_hidden_units=(16, 8),
                                                                  **zero_l2)), x, y, 74)

    mkv, xv, yv = _varlen_case(rng)
    GF.model_case("ifm_varlen", "IFM", GP._columns(mkv, dict(dnn_hidden_units=(8,), **zero_l2)), xv, yv, 75)
    GF.model_case("difm_two_heads_varlen", "DIFM",
                  GP._columns(mkv, dict(att_embedding_size=4, att_head_num=2, dnn_hidden_units=(16, 8), **zero_l2)),
                  xv, yv, 76)


def builders():
    import golden_models as G
    import generate_builders as GB
    from test_reference_builders_dropin import signature, builder_args
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
        for b in ("IFM", "DIFM"):
            sig = inspect.signature(GB._reference_builder(os.path.join(REF, "deepctr"), b))
            out["defaults"][b] = [[k, repr(p.default)] for k, p in sig.parameters.items()]
    E.clear_session()
    with open(BUILDERS_JSON, "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
    print("wrote", os.path.basename(BUILDERS_JSON), sorted(out["signatures"]))


if __name__ == "__main__":
    fixtures()
    builders()
