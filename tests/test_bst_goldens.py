"""The BST fixtures made by the reference's own code (tests/golden/generate_bst.py).

Model fixtures: model_golden_checks' checks (shared by every fixture family), bound below; on the GPU,
test_model_fixture_gpu is the one-SGD-step check.
CPU: the restatement of tests/bst_oracle.py reproduces every layer fixture (outputs and all gradients).
GPU: the Transformer / PositionEncoding / LayerNormalization layers reproduce the fixtures in both GEMM precisions:
outputs and gradients.
"""
import glob
import json
import os

import numpy as np
import pytest
import torch

import b2_helpers as H
import bst_oracle as BO
import model_golden_checks as C

HERE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
LAYERS = os.path.join(HERE, "bst")
LAYER_CASES = sorted(os.path.basename(p)[:-4] for p in glob.glob(os.path.join(LAYERS, "*.npz")))

T = C.model_tests("bst")
test_fixture_sets = T.fixture_set
test_oracle_reproduces_model_fixture = T.oracle
test_builder_creates_the_reference_weight_set = T.weight_set
test_builder_carries_the_fixture_weights_and_the_reference_graph = T.graph
test_reference_default_arguments_are_the_same = T.defaults
T = C.gpu_model_tests("bst")
test_model_forward_matches_reference = T.forward
test_model_fixture_gpu = T.sgd_step


def _layer(name):
    d = np.load(os.path.join(LAYERS, name + ".npz"))
    meta = json.loads(str(d["meta"]))
    xs = [d["x_%d" % i] for i in range(len([k for k in d.files if k.startswith("x_")]))]
    return d, meta, xs


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
    H.close(out.detach().numpy(), d["out"], "out", 1e-5)
    (out * torch.as_tensor(d["dout"])).sum().backward()
    for i, t in enumerate(ts):
        if "gx_%d" % i in d.files:
            H.close(t.grad.numpy(), d["gx_%d" % i], "gx_%d" % i, 1e-4)
    for k, t in W.items():
        if "g_" + k in d.files:
            g = t.grad.numpy() if t.grad is not None else np.zeros_like(d["g_" + k])
            H.close(g, d["g_" + k], k, 1e-4) if np.abs(d["g_" + k]).max() > 0 else \
                np.testing.assert_array_equal(g, 0)


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
    H.close(E.contiguous(y).cpu().numpy(), d["out"], "out", tol)
    y.requires_grad = True
    E.add_grad(y, torch.tensor(d["dout"], device=cuda))
    tape.backward()
    for i, v in enumerate(vs):
        if "gx_%d" % i in d.files:
            H.close(v.grad.cpu().numpy().reshape(d["gx_%d" % i].shape), d["gx_%d" % i], "gx_%d" % i, tol)
    for k, w in mine.items():
        if "g_" + k in d.files and np.abs(d["g_" + k]).max() > 0:
            H.close(w.grad.cpu().numpy(), d["g_" + k], k, tol)
