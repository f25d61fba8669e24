#!/usr/bin/env python
"""Generate tests/golden/*.npz by executing the REFERENCE's unmodified layer code
(/root/reference/deepctr/layers/*.py) under the torch-backed ``tensorflow`` stand-in of
tf_torch_shim.py.  Run in the build container (needs /root/reference); the fixtures are committed so
the GPU test machine, which has no reference tree, can check both the oracle and the CUDA path against them.

    python tests/golden/generate.py

Every fixture holds the layer's constructor arguments (json), the input arrays ``in_<i>``, optional
``mask`` / ``training``, the weights ``w_<name>`` exactly as the reference layer created and named
them, and the reference output ``out``.
"""
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

import tf_torch_shim as S  # noqa: E402


def _set_random_weights(layer, rng, scale=0.4):
    """Overwrite every weight (recursively through sub-layers) in place so values are O(1)."""
    seen = []

    def visit(l):
        for name, t in l._w:
            if "moving" in name:
                continue
            t.copy_(torch.as_tensor(rng.normal(0, scale, size=tuple(t.shape)).astype(np.float32)))
            seen.append((l, name, t))
        for v in vars(l).values():
            vs = v if isinstance(v, (list, tuple)) else [v]
            for e in vs:
                if isinstance(e, S.Layer) and e is not l:
                    visit(e)

    visit(layer)
    return seen


def _collect(layer, prefix=""):
    out = {}
    for name, t in layer._w:
        out[prefix + name] = t.numpy().copy()
    for key, v in vars(layer).items():
        vs = v if isinstance(v, (list, tuple)) else [v]
        for i, e in enumerate(vs):
            if isinstance(e, S.Layer) and e is not layer:
                sub = "%s%s%s/" % (prefix, key, "" if not isinstance(v, (list, tuple)) else str(i))
                out.update(_collect(e, sub))
                if isinstance(e, S.BatchNormalization) and e.moving_mean is not None:
                    out[sub + "moving_mean"] = e.moving_mean.numpy().copy()
                    out[sub + "moving_variance"] = e.moving_variance.numpy().copy()
    return out


def save(name, cls, kwargs, inputs, out, weights, extra=None):
    d = {"meta": np.array(json.dumps({"layer": cls, "kwargs": kwargs, "extra": extra or {}}))}
    for i, a in enumerate(inputs):
        d["in_%d" % i] = np.asarray(a)
    for k, v in weights.items():
        d["w_" + k] = v
    d["out"] = out.detach().numpy() if isinstance(out, torch.Tensor) else np.asarray(out)
    np.savez(os.path.join(HERE, name + ".npz"), **d)
    print("%-44s out%s" % (name, tuple(d["out"].shape)))


def run(L, name, cls, kwargs, inputs, rng, call_kwargs=None, build_first=True, scale=0.4):
    layer = getattr(L, cls)(**kwargs)
    tin = [torch.as_tensor(a) for a in inputs]
    arg = tin[0] if len(tin) == 1 else tin
    layer.build(S._shape_of(arg))
    layer.built = True
    # sub-layers (DNN inside LocalActivationUnit, Dice inside DNN) are built lazily by the shim's
    # __call__: run once to create them, then randomise everything and run again for the record
    layer.call(arg, **(call_kwargs or {}))
    _set_random_weights(layer, rng, scale)
    for l in [layer]:
        pass
    out = layer.call(arg, **(call_kwargs or {}))
    extra = {k: (v.numpy().tolist() if isinstance(v, torch.Tensor) else
                 ([m.numpy().tolist() if m is not None else None for m in v] if isinstance(v, list) else v))
             for k, v in (call_kwargs or {}).items()}
    save(name, cls, kwargs, inputs, out, _collect(layer), extra)


def main():
    L = S.install()
    rng = np.random.RandomState(20260922)
    f32 = np.float32
    x3 = rng.normal(size=(5, 4, 3)).astype(f32)                     # tests/layers/interaction_test.py:11-14
    run(L, "fm", "FM", {}, [x3], rng)
    x2 = rng.normal(size=(6, 7)).astype(f32)
    run(L, "crossnet_vector2", "CrossNet", {"layer_num": 2, "parameterization": "vector"}, [x2], rng)
    run(L, "crossnet_matrix1", "CrossNet", {"layer_num": 1, "parameterization": "matrix"}, [x2], rng)
    run(L, "crossnet_vector0", "CrossNet", {"layer_num": 0}, [x2], rng)
    run(L, "cin_10_8_split", "CIN", {"layer_size": (10, 8), "split_half": True, "activation": "relu"}, [x3], rng)
    run(L, "cin_10_nosplit", "CIN", {"layer_size": (10,), "split_half": False, "activation": "relu"}, [x3], rng)
    run(L, "cin_8_6_5_linear", "CIN", {"layer_size": (8, 6, 5), "split_half": False, "activation": "linear"},
        [x3], rng)
    run(L, "interacting_h2_res", "InteractingLayer", {"att_embedding_size": 5, "head_num": 2, "use_res": True},
        [x3], rng)
    run(L, "interacting_h1_nores_scaled", "InteractingLayer",
        {"att_embedding_size": 4, "head_num": 1, "use_res": False, "scaling": True}, [x3], rng)
    # sequences: B=4, T=10, E=8 (tests/layers/sequence_test.py:17-19)
    B, T, E = 4, 10, 8
    seq = rng.normal(size=(B, T, E)).astype(f32)
    lens = np.array([[0], [3], [10], [7]], dtype=np.int32)
    mask = torch.as_tensor(np.arange(T)[None, :] < lens)
    for mode in ("sum", "mean", "max"):
        run(L, "seqpool_%s_len" % mode, "SequencePoolingLayer", {"mode": mode, "supports_masking": False},
            [seq, lens], rng)
        run(L, "seqpool_%s_mask" % mode, "SequencePoolingLayer", {"mode": mode, "supports_masking": True},
            [seq], rng, call_kwargs={"mask": mask})
    w = rng.rand(B, T, 1).astype(f32)
    lens1 = np.array([[1], [3], [10], [7]], dtype=np.int32)
    for norm in (True, False):
        run(L, "weightedseq_norm%d_len" % norm, "WeightedSequenceLayer",
            {"weight_normalization": norm, "supports_masking": False}, [seq, lens1, w], rng)
    run(L, "weightedseq_norm1_mask", "WeightedSequenceLayer", {"weight_normalization": True, "supports_masking": True},
        [seq, w], rng, call_kwargs={"mask": [torch.as_tensor(np.arange(T)[None, :] < lens1), None]})
    q = rng.normal(size=(B, 1, E)).astype(f32)
    for act in ("sigmoid", "dice"):
        for wn in (False, True):
            run(L, "din_att_%s_wn%d_len" % (act, wn), "AttentionSequencePoolingLayer",
                {"att_hidden_units": (6, 5), "att_activation": act, "weight_normalization": wn}, [q, seq, lens1], rng)
    run(L, "din_att_sigmoid_mask", "AttentionSequencePoolingLayer",
        {"att_hidden_units": (6, 5), "att_activation": "sigmoid", "supports_masking": True}, [q, seq], rng,
        call_kwargs={"mask": [None, torch.as_tensor(np.arange(T)[None, :] < lens1)]})
    run(L, "din_att_score", "AttentionSequencePoolingLayer",
        {"att_hidden_units": (6, 5), "att_activation": "sigmoid", "return_score": True, "weight_normalization": True},
        [q, seq, lens1], rng)
    run(L, "lau_sigmoid", "LocalActivationUnit", {"hidden_units": (6, 5), "activation": "sigmoid"}, [q, seq], rng)
    xd = rng.normal(size=(9, 11)).astype(f32)
    run(L, "dnn_relu", "DNN", {"hidden_units": (7, 5), "activation": "relu"}, [xd], rng)
    run(L, "dnn_dice_infer", "DNN", {"hidden_units": (7, 5), "activation": "dice"}, [xd], rng,
        call_kwargs={"training": False})
    run(L, "dnn_dice_train", "DNN", {"hidden_units": (7, 5), "activation": "dice"}, [xd], rng,
        call_kwargs={"training": True})
    run(L, "dnn_outact", "DNN", {"hidden_units": (7, 5), "activation": "relu", "output_activation": "sigmoid"},
        [xd], rng)
    run(L, "dice_train", "Dice", {}, [xd], rng, call_kwargs={"training": True})
    z = rng.normal(size=(12, 1)).astype(f32)
    run(L, "prediction_binary", "PredictionLayer", {"task": "binary"}, [z], rng)
    run(L, "prediction_regression", "PredictionLayer", {"task": "regression"}, [z], rng)
    sp = rng.normal(size=(8, 1, 6)).astype(f32)
    dn = rng.normal(size=(8, 4)).astype(f32)
    run(L, "linear_mode0", "Linear", {"mode": 0}, [sp], rng)
    run(L, "linear_mode1", "Linear", {"mode": 1, "use_bias": True}, [dn], rng)
    run(L, "linear_mode2", "Linear", {"mode": 2, "use_bias": True}, [sp, dn], rng)
    # the reference's only known-answer vector, through its own Hash layer + vocabulary file
    vocab = os.path.join("/root/reference", "tests", "layers", "vocabulary_example.csv")
    h = L.Hash(num_buckets=4, vocabulary_path=vocab)
    out = h.call(S.constant([["lake"], ["johnson"], ["lakemerson"]]))
    assert out.numpy().tolist() == [[1], [3], [0]], out      # tests/layers/utils_test.py:20-22
    np.savez(os.path.join(HERE, "hash_vocab_kat.npz"), keys=np.array(["lake", "johnson", "lakemerson"]),
             out=out.numpy(), vocab=np.array(open(vocab).read()))
    print("hash_vocab_kat                               out", out.numpy().tolist())


if __name__ == "__main__":
    main()
