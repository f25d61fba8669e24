"""The BST fixtures made by the reference's own code (tests/golden/generate_bst.py).

CPU: the restatement of tests/bst_oracle.py reproduces every layer and model fixture (outputs, loss, all gradients);
deepctr_b200's BST builds the graph the reference's bst.py source builds on this package, carries the fixtures'
weights by name, and has the reference's keyword defaults.
GPU: the Transformer / PositionEncoding / LayerNormalization layers and the BST models reproduce the fixtures in both
GEMM precisions: outputs and gradients, logits and predictions within 1e-4, one SGD step's weight updates.
"""
import glob
import json
import os

import numpy as np
import pytest
import torch

import bst_oracle as BO
import golden_models as G

HERE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
LAYERS = os.path.join(HERE, "bst")
MODELS_BST = os.path.join(HERE, "models_bst")
LAYER_CASES = sorted(os.path.basename(p)[:-4] for p in glob.glob(os.path.join(LAYERS, "*.npz")))
MODEL_CASES = sorted(os.path.basename(p)[:-4] for p in glob.glob(os.path.join(MODELS_BST, "*.npz")))
BUILDERS_JSON = os.path.join(HERE, "reference_builders_bst.json")


class Fixture(G.Fixture):
    def __init__(self, name):
        saved, G.MODELS = G.MODELS, MODELS_BST
        try:
            G.Fixture.__init__(self, name)
        finally:
            G.MODELS = saved


def builder_args(fx):
    from deepctr_b200 import feature_column as FC
    kw = dict(fx.kwargs)
    if "dnn_hidden_units" in kw:
        kw["dnn_hidden_units"] = tuple(kw["dnn_hidden_units"])
    return (G.columns(fx, "dnn", FC), ["item_id", "cate_id"]), kw


def weight_map(fx, model):
    return G.weight_map(fx, model)


def _layer(name):
    d = np.load(os.path.join(LAYERS, name + ".npz"))
    meta = json.loads(str(d["meta"]))
    xs = [d["x_%d" % i] for i in range(len([k for k in d.files if k.startswith("x_")]))]
    return d, meta, xs


def _close(got, want, what, rtol=1e-4):
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    scale = max(float(np.abs(want).max()), 1e-12)
    err = float(np.abs(got - want).max()) / scale
    assert err < rtol, "%s: max error %.3e relative to max |value|" % (what, err)


# ---- CPU: the oracle reproduces the fixtures ----------------------------------------------------------------
def _oracle_layer(meta, xs, W, d):
    kw = meta["kwargs"]
    cls = meta["layer"]
    if cls == "LayerNormalization":
        return BO.layer_norm(xs[0], W["gamma"], W["beta"])
    if cls == "PositionEncoding":
        return BO.position_encoding(xs[0], W["lookup_table"], kw.get("scale", True))
    T = xs[0].shape[1]
    if meta["masked"]:
        qv, kv = torch.as_tensor(d["mask_0"]), torch.as_tensor(d["mask_1"])
    else:
        ar = torch.arange(T)[None, :]
        qv, kv = ar < torch.as_tensor(xs[2]).long(), ar < torch.as_tensor(xs[3]).long()
    return BO.transformer(xs[0], xs[1], qv, kv, W, **kw)


@pytest.mark.parametrize("name", LAYER_CASES)
def test_oracle_reproduces_layer_fixture(name):
    d, meta, xs = _layer(name)
    ts = [torch.tensor(a, requires_grad=a.dtype == np.float32) for a in xs]
    W = {k[2:]: torch.tensor(d[k], requires_grad=True) for k in d.files if k.startswith("w_")}
    out = _oracle_layer(meta, ts, W, d)
    _close(out.detach().numpy(), d["out"], "out", 1e-5)
    (out * torch.as_tensor(d["dout"])).sum().backward()
    for i, t in enumerate(ts):
        if "gx_%d" % i in d.files:
            _close(t.grad.numpy(), d["gx_%d" % i], "gx_%d" % i, 1e-4)
    for k, t in W.items():
        if "g_" + k in d.files:
            g = t.grad.numpy() if t.grad is not None else np.zeros_like(d["g_" + k])
            _close(g, d["g_" + k], k, 1e-4) if np.abs(d["g_" + k]).max() > 0 else \
                np.testing.assert_array_equal(g, 0)


def oracle_weights(fx):
    leaves = {k: torch.tensor(v, requires_grad=True) for k, v in fx.w.items()}
    tables = {k.split("/")[0][len("sparse_emb_"):]: v for k, v in leaves.items() if k.endswith("/embeddings")}
    trs = []
    for name in fx.layer_names("Transformer"):
        trs.append({k[len(name) + 1:]: v for k, v in leaves.items() if k.startswith(name + "/")})
    p = fx.layer_names("AttentionSequencePoolingLayer")[0] + "/local_att/"
    n = len([k for k in leaves if k.startswith(p + "dnn/kernel")])
    lau = {"dnn_kernels": [leaves["%sdnn/kernel%d" % (p, i)] for i in range(n)],
           "dnn_biases": [leaves["%sdnn/bias%d" % (p, i)] for i in range(n)],
           "kernel": leaves[p + "kernel"], "bias": leaves[p + "bias"]}
    dnn = [nm for nm in fx.layer_names("DNN")][-1]
    m = len([k for k in leaves if k.startswith(dnn + "/kernel")])
    W = {"tables": tables, "transformers": trs, "lau": lau,
         "dnn_kernels": [leaves["%s/kernel%d" % (dnn, i)] for i in range(m)],
         "dnn_biases": [leaves["%s/bias%d" % (dnn, i)] for i in range(m)],
         "dense_kernel": leaves[fx.layer_names("Dense")[-1] + "/kernel"],
         "global_bias": leaves[fx.layer_names("PredictionLayer")[-1] + "/global_bias"]}
    return W, leaves


def oracle_forward(fx, W):
    from deepctr_b200 import feature_column as FC
    kw = fx.kwargs
    return BO.bst(fx.inputs(), G.columns(fx, "dnn", FC), ["item_id", "cate_id"], W,
                  transformer_num=kw.get("transformer_num", 1), att_head_num=kw.get("att_head_num", 8))


@pytest.mark.parametrize("name", MODEL_CASES)
def test_oracle_reproduces_model_fixture(name):
    from oracle import ops as O
    fx = Fixture(name)
    W, leaves = oracle_weights(fx)
    logit, pred = oracle_forward(fx, W)
    _close(logit.detach().numpy(), fx.logit, "logit", 1e-5)
    _close(pred.detach().numpy(), fx.out, "out", 1e-5)
    loss = O.binary_crossentropy(fx.y, pred)
    assert abs(float(loss.detach()) - fx.loss) < 1e-5 * max(1.0, abs(fx.loss))
    loss.backward()
    for k, t in leaves.items():
        if k in fx.g and np.abs(fx.g[k]).max() > 0:
            _close(t.grad.numpy(), fx.g[k], k, 1e-4)


@pytest.mark.parametrize("name", MODEL_CASES)
def test_builder_carries_the_fixture_weights_and_the_reference_graph(name):
    from deepctr_b200 import engine as E, models as M
    import test_reference_builders_dropin as D
    fx = Fixture(name)
    args, kw = builder_args(fx)
    E.clear_session()
    model = M.BST(*args, **kw)
    weight_map(fx, model)
    with open(BUILDERS_JSON) as f:
        ref = json.load(f)
    a, b = ref["signatures"][name], D.signature(model)
    assert a["inputs"] == b["inputs"] and a["weights"] == b["weights"]
    assert a["slots"] == b["slots"] and a["fast"] == b["fast"]
    assert sorted(a["layers"]) == sorted(b["layers"])


def test_reference_default_arguments_are_the_same():
    import inspect
    from deepctr_b200 import models as M
    with open(BUILDERS_JSON) as f:
        ref = json.load(f)["defaults"]["BST"]
    mine = inspect.signature(M.BST)
    assert [k for k, _ in ref] == list(mine.parameters)
    for k, dflt in ref:
        assert dflt == repr(mine.parameters[k].default), k


# ---- GPU: the CUDA layers and models reproduce the fixtures ----------------------------------------------
@pytest.mark.gpu
@pytest.mark.usefixtures("gemm_precision")
@pytest.mark.parametrize("name", LAYER_CASES)
def test_layer_fixture_gpu(cuda, name):
    from deepctr_b200 import engine as E, layers as Lyr
    d, meta, xs = _layer(name)
    E.clear_session()
    layer = getattr(Lyr, meta["layer"])(**meta["kwargs"])
    vs = []
    for i, a in enumerate(xs):
        v = E.Var(torch.tensor(a, device=cuda), requires_grad=a.dtype == np.float32)
        if meta["masked"]:
            v.mask = E.KMask(lengths=torch.tensor(d["mask_%d" % i].sum(1).astype(np.int32), device=cuda),
                             maxlen=a.shape[1])
        vs.append(v)
    ins = vs if len(vs) > 1 else vs[0]
    layer._maybe_build(E._shape_of(ins))
    mine = {w.name.split("/", 1)[1]: w for w in layer.weights}
    assert sorted(mine) == sorted(k[2:] for k in d.files if k.startswith("w_")), name
    for k, w in mine.items():
        w.set_value(d["w_" + k])
        w.materialize()
    tape = E.Tape()
    with E.recording(tape):
        y = layer._invoke(ins, False)
    tol = 2e-4
    _close(E.contiguous(y).cpu().numpy(), d["out"], "out", tol)
    y.requires_grad = True
    E.add_grad(y, torch.tensor(d["dout"], device=cuda))
    tape.backward()
    for i, v in enumerate(vs):
        if "gx_%d" % i in d.files:
            _close(v.grad.cpu().numpy().reshape(d["gx_%d" % i].shape), d["gx_%d" % i], "gx_%d" % i, tol)
    for k, w in mine.items():
        if "g_" + k in d.files and np.abs(d["g_" + k]).max() > 0:
            _close(w.grad.cpu().numpy(), d["g_" + k], k, tol)


@pytest.mark.gpu
@pytest.mark.usefixtures("gemm_precision")
@pytest.mark.parametrize("name", MODEL_CASES)
def test_model_fixture_gpu(cuda, name):
    from deepctr_b200 import engine as E, models as M
    from deepctr_b200.engine import SGD
    fx = Fixture(name)
    args, kw = builder_args(fx)
    E.clear_session()
    model = M.BST(*args, **kw)
    wm = G.assign_weights(fx, model)
    x = fx.inputs()
    np.testing.assert_allclose(model.predict(x, batch_size=len(fx.y)), fx.out, rtol=1e-4, atol=1e-5)
    lr = 0.5
    model.compile(SGD(lr), "binary_crossentropy", embedding_update="dense")
    loss = model.train_on_batch(x, fx.y)
    assert abs(loss - fx.loss) <= 2e-4 * max(1.0, abs(fx.loss)), (loss, fx.loss)
    for key, w in wm.items():
        if key not in fx.g:
            continue
        want = fx.g[key]
        got = (fx.w[key] - w.value()) / lr
        np.testing.assert_allclose(got, want, rtol=2e-3, atol=3e-4 * float(np.abs(want).max()) + 2e-6, err_msg=key)
