#!/usr/bin/env python
"""Generate the BST fixtures (the builder and its Transformer / PositionEncoding / LayerNormalization layers) from the
REFERENCE's own, unmodified deepctr/layers/sequence.py, deepctr/layers/normalization.py and
deepctr/models/sequence/bst.py, executed eagerly under the torch-backed ``tensorflow`` stand-in of tf_torch_shim.py
(the recipe of generate_fibinet.py).  The few TensorFlow symbols these files need beyond the shim are stood in for
here, so that tf_torch_shim.py - and with it every existing fixture - stays as it is.

    python tests/golden/generate_bst.py          (build container only: needs the reference checkout)

Writes
  tests/golden/bst/*.npz                    layer level: ``meta``, the inputs ``x_<i>`` (float inputs get ``gx_<i>``),
                                            every weight ``w_<name>`` (nested layers by attribute: ``ln/gamma``), the
                                            output ``out``, an upstream gradient ``dout`` and the gradients ``g_<name>``;
  tests/golden/models_bst/*.npz             model level, the layout of tests/golden/models/;
  tests/golden/reference_builders_bst.json  the graphs the reference's bst.py SOURCE FILE builds on this package for
                                            those fixtures, and its keyword defaults.
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
from generate_models import _col_meta, _collect  # noqa: E402

REF = "/root/reference"
LAYER_OUT = os.path.join(HERE, "bst")
MODEL_OUT = os.path.join(HERE, "models_bst")
BUILDERS_JSON = os.path.join(HERE, "reference_builders_bst.json")


class _Shape(tuple):
    def as_list(self):
        return list(self)


def _matrix_set_diag(x, diag):
    n = min(x.shape[-2], x.shape[-1])
    eye = torch.eye(x.shape[-2], x.shape[-1], dtype=torch.bool)
    d = torch.zeros_like(x)
    d[..., torch.arange(n), torch.arange(n)] = diag[..., :n]
    return torch.where(eye, d, x)


def install():
    """The shim plus what the Transformer / PositionEncoding / LayerNormalization code needs."""
    S.install(REF)
    torch.Tensor.get_shape = lambda self: _Shape(self.shape)
    # TF tensors are immutable: `outputs -= reduce_max(...)` (sequence.py:600) and the like rebind the name
    torch.Tensor.__iadd__ = lambda self, o: self + o
    torch.Tensor.__isub__ = lambda self, o: self - o
    torch.Tensor.__imul__ = lambda self, o: self * o
    torch.Tensor.__itruediv__ = lambda self, o: self / o
    tf = sys.modules["tensorflow"]
    tf.equal = lambda x, y, **kw: x == y
    tf.shape = lambda x, **kw: list(x.shape)
    tf.range = lambda n, **kw: torch.arange(int(n))
    tf.nn.embedding_lookup = lambda params, ids, **kw: params[ids.to(torch.int64)]
    tf.compat = S._mod("tensorflow.compat")
    tf.compat.v1 = S._mod("tensorflow.compat.v1", matrix_set_diag=_matrix_set_diag)
    K = sys.modules["tensorflow.keras.backend"]
    K.mean = lambda x, axis=None, keepdims=False: torch.mean(x, dim=axis, keepdim=keepdims)
    K.sqrt = torch.sqrt
    K.square = lambda x: x * x
    importlib.import_module("deepctr.feature_column")
    importlib.import_module("deepctr.layers.sequence")


def layer_case(name, cls, kwargs, inputs, seed, masks=None, module="deepctr.layers.sequence"):
    """inputs: list of numpy arrays (float: differentiated); masks: Keras masks for supports_masking=True."""
    S.CTX.reset()
    S.CTX.rng = np.random.RandomState(seed)
    S.CTX.grad = True
    ts = []
    for a in inputs:
        t = torch.tensor(a, requires_grad=a.dtype == np.float32)
        ts.append(t)
    if masks is not None:
        for t, m in zip(ts, masks):
            t._keras_mask = torch.as_tensor(m)
    layer = getattr(sys.modules[module], cls)(**kwargs)
    out = layer(ts if len(ts) > 1 else ts[0])
    rng = np.random.RandomState(seed + 1000)
    dout = rng.normal(0, 1.0, size=tuple(out.shape)).astype(np.float32)
    weights = _collect(layer, "")
    leaves = [t for _, t in weights if t.requires_grad]
    fl = [t for t in ts if t.requires_grad]
    grads = torch.autograd.grad((out * torch.as_tensor(dout)).sum(), fl + leaves, allow_unused=True)
    d = {"meta": np.array(json.dumps({"layer": cls, "kwargs": kwargs, "masked": masks is not None})),
         "out": out.detach().numpy(), "dout": dout}
    gi = iter(grads[:len(fl)])
    for i, (a, t) in enumerate(zip(inputs, ts)):
        d["x_%d" % i] = a
        if t.requires_grad:
            d["gx_%d" % i] = next(gi).numpy()
        if masks is not None:
            d["mask_%d" % i] = np.asarray(masks[i])
    gw = {id(t): g for t, g in zip(leaves, grads[len(fl):])}
    for wn, t in weights:
        d["w_" + wn] = t.detach().numpy().copy()
        if t.requires_grad:
            g = gw.get(id(t))
            d["g_" + wn] = (g if g is not None else torch.zeros_like(t)).numpy()
    np.savez_compressed(os.path.join(LAYER_OUT, name + ".npz"), **d)
    print("%-28s out%s  %d weights" % (name, tuple(d["out"].shape), len(weights)))


def din_batch(FC):
    """tests/models/DIN_test.py:get_xy_fd(hash_flag=True) of the reference (its BST_test.py batch)."""
    cols = [FC.SparseFeat('user', 3, embedding_dim=10), FC.SparseFeat('gender', 2, embedding_dim=4),
            FC.SparseFeat('item_id', 3 + 1, embedding_dim=8), FC.SparseFeat('cate_id', 2 + 1, embedding_dim=4),
            FC.DenseFeat('pay_score', 1)]
    cols += [FC.VarLenSparseFeat(FC.SparseFeat('hist_item_id', vocabulary_size=3 + 1, embedding_dim=8,
                                               embedding_name='item_id'), maxlen=4, length_name="seq_length"),
             FC.VarLenSparseFeat(FC.SparseFeat('hist_cate_id', 2 + 1, embedding_dim=4, embedding_name='cate_id'),
                                 maxlen=4, length_name="seq_length")]
    return cols


def din_batch_x():
    x = {'user': np.array([0, 1, 2]), 'gender': np.array([0, 1, 0]), 'item_id': np.array([1, 2, 3]),
         'cate_id': np.array([1, 2, 2]), 'pay_score': np.array([0.1, 0.2, 0.3], np.float32),
         'hist_item_id': np.array([[1, 2, 3, 0], [3, 2, 1, 0], [1, 2, 0, 0]]),
         'hist_cate_id': np.array([[1, 2, 2, 0], [2, 2, 1, 0], [1, 2, 0, 0]]),
         'seq_length': np.array([3, 3, 2])}
    return {k: (v.astype(np.int32) if v.dtype.kind == "i" else v) for k, v in x.items()}, np.array([1, 0, 1],
                                                                                                np.float32)


def wide_batch(rng, n, T, V=(30, 12), dims=(48, 16)):
    def mk(FC):
        cols = [FC.SparseFeat('user', 7, embedding_dim=8), FC.SparseFeat('item_id', V[0] + 1, embedding_dim=dims[0]),
                FC.SparseFeat('cate_id', V[1] + 1, embedding_dim=dims[1]), FC.DenseFeat('pay_score', 1)]
        cols += [FC.VarLenSparseFeat(FC.SparseFeat('hist_item_id', V[0] + 1, embedding_dim=dims[0],
                                                   embedding_name='item_id'), maxlen=T, length_name="seq_length"),
                 FC.VarLenSparseFeat(FC.SparseFeat('hist_cate_id', V[1] + 1, embedding_dim=dims[1],
                                                   embedding_name='cate_id'), maxlen=T, length_name="seq_length")]
        return cols
    ln = rng.randint(0, T + 1, size=n).astype(np.int32)
    ln[:3] = [0, 1, T]
    pos = np.arange(T)[None, :] < ln[:, None]
    x = {'user': rng.randint(0, 7, n).astype(np.int32), 'item_id': rng.randint(1, V[0] + 1, n).astype(np.int32),
         'cate_id': rng.randint(1, V[1] + 1, n).astype(np.int32), 'pay_score': rng.rand(n).astype(np.float32),
         'hist_item_id': (rng.randint(1, V[0] + 1, (n, T)) * pos).astype(np.int32),
         'hist_cate_id': (rng.randint(1, V[1] + 1, (n, T)) * pos).astype(np.int32), 'seq_length': ln}
    y = (rng.rand(n) < 0.4).astype(np.float32)
    return mk, x, y


def _bst_args(mk, kw):
    def f(FC):
        cols = mk(FC)
        meta = [_col_meta(c, FC) for c in cols]
        return (cols, ['item_id', 'cate_id']), dict(kw), {"linear": meta, "dnn": meta}
    return f


MODEL_CASES = []


def fixtures():
    install()
    for d in (LAYER_OUT, MODEL_OUT):
        if os.path.isdir(d):
            shutil.rmtree(d)
        os.makedirs(d)
    rng = np.random.RandomState(20261016)
    B, T, E = 16, 7, 8
    xq = rng.normal(size=(B, T, E)).astype(np.float32)
    xk = rng.normal(size=(B, T, E)).astype(np.float32)
    ql = np.array([[0], [1], [T]] + [[rng.randint(0, T + 1)] for _ in range(B - 3)], np.int32)
    kl = np.array([[T], [0], [1]] + [[rng.randint(0, T + 1)] for _ in range(B - 3)], np.int32)
    # ---- layers ---------------------------------------------------------------------------------------
    bst_kw = dict(att_embedding_size=4, head_num=2, use_positional_encoding=True, use_res=True, use_feed_forward=True,
                  use_layer_norm=True, blinding=False, supports_masking=False, output_type=None)
    layer_case("transformer_bst_t7_e8_h2", "Transformer", bst_kw, [xq, xk, ql, kl], 1)
    layer_case("transformer_reftest_e8_h8", "Transformer",
               dict(att_embedding_size=1, head_num=8, use_layer_norm=True, output_type='sum', dropout_rate=0.0),
               [xq, xk, ql, kl], 2)
    layer_case("transformer_defaults_e8_h4", "Transformer", dict(att_embedding_size=2, head_num=4),
               [xq, xk, ql, kl], 3)
    qm = np.arange(T)[None, :] < ql
    km = np.arange(T)[None, :] < kl
    layer_case("transformer_masking_e8_h2", "Transformer",
               dict(att_embedding_size=4, head_num=2, use_layer_norm=True, supports_masking=True, output_type=None),
               [xq, xk], 4, masks=[qm, km])
    layer_case("position_encoding", "PositionEncoding", {}, [xq], 5)
    layer_case("position_encoding_zero_pad", "PositionEncoding", dict(zero_pad=True, scale=False), [xq], 6)
    layer_case("layer_normalization", "LayerNormalization", {}, [xq * 3 + 1], 7,
               module="deepctr.layers.normalization")

    # ---- models ---------------------------------------------------------------------------------------
    GP.MODEL_OUT = MODEL_OUT
    GP.MODULES["BST"] = "deepctr.models.sequence.bst"
    x, y = din_batch_x()
    base = dict(dnn_hidden_units=(16, 8), l2_reg_embedding=0)
    cases = [("bst_ref_batch", din_batch, x, y, dict(att_head_num=4, **base)),
             ("bst_two_layers", din_batch, x, y, dict(att_head_num=2, transformer_num=2, **base)),
             ("bst_no_dnn", din_batch, x, y, dict(att_head_num=4, dnn_hidden_units=(), l2_reg_embedding=0))]
    mk, xw, yw = wide_batch(rng, 24, 12)
    cases.append(("bst_wide_e64_h8", mk, xw, yw, dict(att_head_num=8, **base)))
    for i, (name, mk_, xx, yy, kw) in enumerate(cases):
        GP.model_case(name, "BST", _bst_args(mk_, kw), xx, yy, seed=100 + i)
        MODEL_CASES.append(name)


def builders():
    """The graphs the reference's bst.py SOURCE builds on this package for the model fixtures, and its defaults."""
    import generate_builders as GB
    import golden_models as G
    from deepctr_b200 import engine as E
    out = {"signatures": {}, "defaults": {}}
    GB._FILES["BST"] = ("models/sequence/bst.py", "models.sequence.bst")
    with GB._aliased():
        build = GB._reference_builder(REF + "/deepctr", "BST")
        for name in G.FAMILIES["bst"].cases:
            fx = G.FAMILIES["bst"].fixture(name)
            args, kw = G.builder_args(fx)
            E.clear_session()
            model = build(*args, **kw)
            G.weight_map(fx, model)
            out["signatures"][name] = G.signature(model)
        out["defaults"]["BST"] = [[k, repr(p.default)] for k, p in inspect.signature(build).parameters.items()]
    E.clear_session()
    with open(BUILDERS_JSON, "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)


if __name__ == "__main__":
    fixtures()
    if "--fixtures-only" not in sys.argv:
        builders()
