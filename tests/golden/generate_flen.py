#!/usr/bin/env python
"""Generate the FLEN fixtures (the builder and its FieldWiseBiInteraction layer) from the REFERENCE's own,
unmodified deepctr/feature_column.py, deepctr/inputs.py, deepctr/layers/* (FieldWiseBiInteraction in
interaction.py) and deepctr/models/flen.py, executed eagerly under the torch-backed ``tensorflow`` stand-in of
tf_torch_shim.py (the recipe of generate_edcn.py and generate_ccpm.py).

    python tests/golden/generate_flen.py          (build container only: needs the reference checkout)

The symbols FLEN needs beyond the shim are supplied here, so that tf_torch_shim.py and the other generators (and
with them every existing fixture) stay as they are:
  * ``tf.gather(params, indices, axis)`` (the layer's pair gathers), torch.index_select;
  * an integer ``shape`` in Layer.add_weight (Keras takes ``shape=(embedding_size)``, an int);
  * generate_onn's full Keras BatchNormalization for DNN(use_bn=True), bound where deepctr/layers/core.py imported
    the shim's; the fixture keys name the DNN's ``bn_layers<i>`` ``bn<i>``, as the package's DNN does.
The layer fixtures replace the layer's initial weights (ones, 0.5 and zeros) by random values, so that every term
of the output and of the gradients is exercised.

Writes
  tests/golden/flen/*.npz                   layer level: ``meta``, the inputs ``x_<g>``, every weight ``w_<name>``,
                                            the output ``out``, an upstream gradient ``dout`` and the gradients
                                            ``gx_<g>`` / ``g_<name>``;
  tests/golden/models_flen/*.npz            model level, the layout of tests/golden/models/;
  tests/golden/reference_builders_flen.json the graphs the reference's flen.py SOURCE FILE builds on this package
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
import generate_onn as GO  # noqa: E402
import generate_pairwise as GP  # noqa: E402

REF = GF.REF
LAYER_OUT = os.path.join(HERE, "flen")
MODEL_OUT = os.path.join(HERE, "models_flen")
BUILDERS_JSON = os.path.join(HERE, "reference_builders_flen.json")
FILES = {"FLEN": ("models/flen.py", "models.flen")}
# examples/run_flen.py's field_info: the group of each of its 21 sparse features, in its sparse_features order
RUN_FLEN_FIELDS = (("hour", "context"), ("C1", "user"), ("banner_pos", "context"), ("site_id", "context"),
                   ("site_domain", "context"), ("site_category", "context"), ("app_id", "item"),
                   ("app_domain", "item"), ("app_category", "item"), ("device_id", "user"),
                   ("device_model", "user"), ("device_type", "user"), ("device_conn_type", "context"),
                   ("C14", "user"), ("C15", "user"), ("C16", "user"), ("C17", "user"), ("C18", "user"),
                   ("C19", "user"), ("C20", "user"), ("C21", "user"))


def _gather(params, indices, axis=0, **kw):
    return torch.index_select(params, axis, torch.as_tensor(list(indices), dtype=torch.long))


def _add_weight(self, name=None, shape=(), *a, **kw):
    """The shim's Layer.add_weight, also taking Keras' integer ``shape`` (the layer's ``shape=(embedding_size)``)."""
    return _SHIM_ADD_WEIGHT(self, name, (shape,) if isinstance(shape, int) else shape, *a, **kw)


_SHIM_ADD_WEIGHT = S.Layer.add_weight


def _install():
    S.install(REF)
    S.Layer.add_weight = _add_weight
    sys.modules["tensorflow"].gather = _gather
    importlib.import_module("deepctr.feature_column")
    sys.modules["deepctr.layers.core"].BatchNormalization = GO.BatchNormalization


def _model_case(name, *args, **kw):
    """generate_fefm.model_case, then the DNN's ``bn_layers<i>`` keys renamed ``bn<i>``."""
    GF.model_case(name, *args, **kw)
    path = os.path.join(MODEL_OUT, name + ".npz")
    d = dict(np.load(path))
    d = {k.replace("/bn_layers", "/bn"): v for k, v in d.items()}
    np.savez_compressed(path, **d)


def layer_case(name, sizes, dim, use_bias, seed, n=6):
    S.CTX.reset()
    S.CTX.rng = np.random.RandomState(seed)
    S.CTX.grad = True
    rng = np.random.RandomState(seed + 1000)
    xs = [rng.normal(0, 0.5, size=(n, f, dim)).astype(np.float32) for f in sizes]
    xt = [torch.tensor(x, requires_grad=True) for x in xs]
    layer = sys.modules["deepctr.layers.interaction"].FieldWiseBiInteraction(use_bias=use_bias)
    layer.build([tuple(x.shape) for x in xs])
    with torch.no_grad():
        for _, t in layer._w:
            t.copy_(torch.tensor(rng.normal(0.3, 0.5, size=tuple(t.shape)).astype(np.float32)))
    out = layer(xt)
    dout = rng.normal(0, 1.0, size=tuple(out.shape)).astype(np.float32)
    leaves = [t for _, t in layer._w]
    grads = torch.autograd.grad((out * torch.as_tensor(dout)).sum(), xt + leaves)
    kwargs = {"use_bias": use_bias}
    d = {"meta": np.array(json.dumps({"layer": "FieldWiseBiInteraction", "kwargs": kwargs}))}
    for i, x in enumerate(xs):
        d["x_%d" % i] = x
    d.update({"out": out.detach().numpy(), "dout": dout})
    for i in range(len(xs)):
        d["gx_%d" % i] = grads[i].numpy()
    for (wn, t), g in zip(layer._w, grads[len(xs):]):
        d["w_" + wn] = t.detach().numpy().copy()
        d["g_" + wn] = g.numpy()
    np.savez_compressed(os.path.join(LAYER_OUT, name + ".npz"), **d)
    print("%-28s out%s  %d weights" % (name, tuple(d["out"].shape), len(layer._w)))


def _grouped(rng, n, groups, dim, n_dense=0, vocab0=20):
    """Sparse features C1.. with the given group names, n_dense dense features I1.."""
    def make(FC):
        cols = [FC.SparseFeat("C%d" % (i + 1), vocab0 + 3 * i, dim, group_name=g) for i, g in enumerate(groups)]
        return cols + [FC.DenseFeat("I%d" % (i + 1), 1) for i in range(n_dense)]
    x = {"C%d" % (i + 1): rng.randint(0, vocab0 + 3 * i, size=n).astype(np.int32) for i in range(len(groups))}
    x.update({"I%d" % (i + 1): rng.rand(n).astype(np.float32) for i in range(n_dense)})
    y = (rng.rand(n) < 0.3).astype(np.float32)
    return make, x, y


def fixtures():
    _install()
    GF.MODULES["FLEN"] = "deepctr.models.flen"
    GF.MODEL_OUT = MODEL_OUT
    for d in (LAYER_OUT, MODEL_OUT):
        if os.path.isdir(d):
            shutil.rmtree(d)
        os.makedirs(d)

    # ---- layers: G in {2, 3, 8}, E in {1, 4, 16}, use_bias both ways, unequal group sizes ---------------------
    layer_case("fwbi_g2_e4_bias", (2, 3), 4, True, 1)
    layer_case("fwbi_g2_e1_nobias", (1, 2), 1, False, 2)
    layer_case("fwbi_g3_e1_bias", (2, 1, 3), 1, True, 3)
    layer_case("fwbi_g3_e16_nobias", (3, 2, 2), 16, False, 4)
    layer_case("fwbi_g8_e4_nobias", (1, 2, 1, 3, 1, 1, 2, 1), 4, False, 5)
    layer_case("fwbi_g8_e16_bias", (2, 1, 1, 2, 1, 3, 1, 1), 16, True, 6)

    rng = np.random.RandomState(20261023)
    n = 32
    zero_l2 = dict(l2_reg_linear=0, l2_reg_embedding=0)
    # ---- the reference test's configuration (tests/models/FLEN_test.py: groups i % 3, 6 dense, E = 2) ----------
    mk, x, y = _grouped(rng, n, [str(i % 3) for i in range(6)], 2, n_dense=6)
    _model_case("flen_reference_test", "FLEN", GP._columns(mk, dict(dnn_hidden_units=(3,), **zero_l2)), x, y, 121)
    # ---- the defaults on 26 interleaved fields; the same fields in contiguous groups ---------------------------
    mk, x, y = _grouped(rng, n, [str(i % 3) for i in range(26)], 4, n_dense=2)
    _model_case("flen_defaults", "FLEN", GP._columns(mk, dict(zero_l2)), x, y, 122)
    mk, x, y = _grouped(rng, n, [str(i * 3 // 9) for i in range(9)], 4, n_dense=1)
    _model_case("flen_contiguous", "FLEN", GP._columns(mk, dict(dnn_hidden_units=(16, 8), **zero_l2)), x, y, 123)
    # ---- unequal group sizes with a one-member group; exactly two groups; eight groups -------------------------
    mk, x, y = _grouped(rng, n, ["a", "b", "b", "c", "b", "c", "b"], 4)
    _model_case("flen_unequal_groups", "FLEN", GP._columns(mk, dict(dnn_hidden_units=(8,), **zero_l2)), x, y, 124)
    mk, x, y = _grouped(rng, n, ["u", "i", "u", "u", "i"], 4, n_dense=2)
    _model_case("flen_two_groups", "FLEN", GP._columns(mk, dict(dnn_hidden_units=(8,), **zero_l2)), x, y, 125)
    mk, x, y = _grouped(rng, n, ["g%d" % (i % 8) for i in range(11)], 4)
    _model_case("flen_eight_groups", "FLEN", GP._columns(mk, dict(dnn_hidden_units=(8,), **zero_l2)), x, y, 126)
    # ---- a mean-pooled VarLenSparseFeat inside a group; a hashed feature ---------------------------------------
    T = 4
    lens = rng.randint(1, T + 1, size=n)
    seq = rng.randint(1, 13, size=(n, T)).astype(np.int32)
    seq[np.arange(T)[None, :] >= lens[:, None]] = 0
    mkg, xg, yv = _grouped(rng, n, ["a", "b", "a", "b"], 4)

    def varlen(FC):
        return mkg(FC) + [FC.VarLenSparseFeat(FC.SparseFeat("S1", 13, 4, group_name="a"), maxlen=T,
                                              combiner="mean")]
    _model_case("flen_varlen", "FLEN", GP._columns(varlen, dict(dnn_hidden_units=(8,), **zero_l2)),
                dict(xg, S1=seq), yv, 127)

    def hashed(FC):
        return mkg(FC) + [FC.SparseFeat("h1", 7, 4, use_hash=True, group_name="b")]
    _model_case("flen_hashed", "FLEN", GP._columns(hashed, dict(dnn_hidden_units=(8,), **zero_l2)),
                dict(xg, h1=rng.randint(0, 1000, size=n).astype(np.int32)), yv, 128)
    # ---- BatchNormalization in the DNN, no DNN, regression ------------------------------------------------------
    mk, x, y = _grouped(rng, n, [str(i % 3) for i in range(6)], 4, n_dense=2)
    _model_case("flen_dnn_bn", "FLEN", GP._columns(mk, dict(dnn_hidden_units=(8,), dnn_use_bn=True, **zero_l2)),
                x, y, 129)
    _model_case("flen_no_dnn", "FLEN", GP._columns(mk, dict(dnn_hidden_units=(), **zero_l2)), x, y, 130)
    yr = rng.normal(0, 1, size=n).astype(np.float32)
    _model_case("flen_regression", "FLEN", GP._columns(mk, dict(dnn_hidden_units=(8,), task="regression",
                                                                **zero_l2)), x, yr, 131, task="regression")
    # ---- examples/run_flen.py's 21 fields in its three groups, E = 16 ------------------------------------------
    def run_flen(FC):
        return [FC.SparseFeat(f, 10 + 2 * i, 16, group_name=g) for i, (f, g) in enumerate(RUN_FLEN_FIELDS)]
    xr = {f: rng.randint(0, 10 + 2 * i, size=n).astype(np.int32) for i, (f, _) in enumerate(RUN_FLEN_FIELDS)}
    _model_case("flen_run_flen_layout", "FLEN", GP._columns(run_flen, dict(dnn_hidden_units=(32, 16), **zero_l2)),
                xr, (rng.rand(n) < 0.3).astype(np.float32), 132)


def builders():
    import golden_models as G
    import generate_builders as GB
    from golden_models import signature, builder_args
    from deepctr_b200 import engine as E
    from deepctr_b200.layers import interaction as LI
    out = {"signatures": {}, "defaults": {}}
    names = sorted(os.path.basename(p)[:-4] for p in os.listdir(MODEL_OUT) if p.endswith(".npz"))
    GB._FILES.update(FILES)
    GP.MODEL_OUT = MODEL_OUT
    with GB._aliased():
        assert sys.modules["refdrop.layers.interaction"].FieldWiseBiInteraction is LI.FieldWiseBiInteraction
        for name in names:
            fx = GP._fixture(name)
            args, kw = builder_args(fx)
            build = GB._reference_builder(os.path.join(REF, "deepctr"), fx.builder)
            E.clear_session()
            model = build(*args, **kw)
            G.weight_map(fx, model)
            out["signatures"][name] = signature(model)
        sig = inspect.signature(GB._reference_builder(os.path.join(REF, "deepctr"), "FLEN"))
        out["defaults"]["FLEN"] = [[k, repr(p.default)] for k, p in sig.parameters.items()]
    E.clear_session()
    with open(BUILDERS_JSON, "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
    print("wrote", os.path.basename(BUILDERS_JSON), sorted(out["signatures"]))


if __name__ == "__main__":
    fixtures()
    builders()
