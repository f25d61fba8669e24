"""Shared test helpers: synthetic CTR data and training runs, GPU logits and tolerances, oracle weights."""
import numpy as np
import torch


def criteo_like(rng, n, n_sparse=6, n_dense=3, vocab=50, dim=8, dtype="int32"):
    from deepctr_b200.feature_column import SparseFeat, DenseFeat
    cols = [SparseFeat("C%d" % i, vocab + i, dim, dtype=dtype) for i in range(n_sparse)]
    cols += [DenseFeat("I%d" % i, 1) for i in range(n_dense)]
    x = {"C%d" % i: rng.randint(0, vocab + i, size=n).astype(np.int32 if dtype == "int32" else np.int64)
         for i in range(n_sparse)}
    x.update({"I%d" % i: rng.rand(n).astype(np.float32) for i in range(n_dense)})
    y = (rng.rand(n) < 0.3).astype(np.float32)
    return cols, x, y


def criteo_model(builder, rng, n_dense=3, **kw):
    """``builder`` over criteo_like's 10 sparse columns (vocabulary 50 + i, dim 8) and ``n_dense`` dense ones, with
    l2 = 0 and seed 3, and a batch of 512 drawn from ``rng``: (model, x, y)."""
    from deepctr_b200 import engine as E, models as M
    cols, x, y = criteo_like(rng, 512, n_sparse=10, n_dense=n_dense)
    E.clear_session()
    if builder == "PNN":                      # PNN(dnn_feature_columns, ...): no linear part
        return M.PNN(cols, l2_reg_embedding=0, seed=3, **kw), x, y
    l2 = "l2_reg_embedding_feat" if builder == "DeepFEFM" else "l2_reg_embedding"
    return getattr(M, builder)(cols, cols, l2_reg_linear=0, seed=3, **{l2: 0}, **kw), x, y


def train(builder, graph, kw, placed=True, steps=6, init=None):
    """``steps`` SGD steps of criteo_model(builder, RandomState(4), **kw), built with the DNN-input placement on or
    off, from ``init`` or from the built model's weights: (losses, {name: weight}, replayed launches, init)."""
    from deepctr_b200 import inputs as I
    from deepctr_b200.engine import SGD
    I.DNN_INPUT_PLACEMENT = placed
    try:
        model, x, y = criteo_model(builder, np.random.RandomState(4), **kw)
    finally:
        I.DNN_INPUT_PLACEMENT = True
    if builder == "FiBiNET":
        assert bool(model.planner.dnn_places) == placed
    elif builder == "PNN":
        products = kw.get("use_inner", True) or kw.get("use_outter", False)
        assert bool(model.planner.pnn_places) == (placed and products)
    if init is None:            # Keras leaves the Dense kernels unseeded: start every run from the same weights
        init = [w.value() for w in model.weights]
    else:
        model.set_weights(init)
    model.compile(SGD(0.05), "binary_crossentropy", embedding_update="sparse", step_graph=graph)
    losses = [model.train_on_batch(x, y) for _ in range(steps)]
    return losses, {w.name: w.value() for w in model.weights}, model.replayed_launches, init


def logits(model, x):
    """pre-activation logits of the compiled graph (what PredictionLayer receives)."""
    from deepctr_b200 import engine as E
    model._materialize()
    feed = model._feed(x)
    logit_t, head = model._head()
    vals = model._run(feed, False, upto=head)
    return E.contiguous(vals[id(logit_t)]).reshape(-1, 1).cpu().numpy()


def logit_tol(want):
    """absolute tolerance of a GPU model's logits or predictions in the current GEMM precision."""
    from deepctr_b200 import ops, _lib as L
    scale = max(float(np.abs(want).max()), 1e-3)
    return (1e-4 if ops.GEMM_PRECISION == L.GEMM_BF16X3 else 2e-5) * scale


def close(got, want, what, tol=2e-5, floor=0.0):
    """Max error relative to max |want|, or to ``floor`` when that is larger: the magnitude of the terms whose
    difference a kernel forms where the result cancels to about 0.  Takes numpy arrays or torch tensors."""
    got, want = torch.as_tensor(got).double(), torch.as_tensor(want).double()
    scale = max(float(want.abs().max()), float(floor), 1e-30)
    err = float((got - want).abs().max()) / scale
    assert err < tol, "%s: max error %.3e relative to max |value|" % (what, err)


def randomize_weights(model, rng, std=0.1):
    """Replace the reference initialisers (zeros / 1e-4) by O(0.1) values so every term of the logit
    carries signal in the parity check."""
    for w in model.weights:
        if w.name.endswith("moving_variance"):
            w.set_value(np.abs(rng.normal(1.0, 0.1, size=w.shape)).astype(np.float32))
        else:
            w.set_value(rng.normal(0, std, size=w.shape).astype(np.float32))


def oracle_weights(model, requires_grad=False):
    """Collect the model's weights in the structure oracle/models.py expects."""
    from deepctr_b200.inputs import Embedding
    from deepctr_b200.layers.core import DNN, PredictionLayer
    from deepctr_b200.layers.interaction import CIN, CrossNet, InteractingLayer
    from deepctr_b200.layers.sequence import AttentionSequencePoolingLayer
    from deepctr_b200.layers.utils import Linear
    from deepctr_b200.engine import Dense

    def t(w):
        return torch.tensor(w.value(), requires_grad=requires_grad)

    W = {"tables": {}, "att": []}
    denses = []
    for l in model.layers:
        if isinstance(l, Embedding):
            W["tables"][l.name] = t(l.embeddings)
        elif isinstance(l, AttentionSequencePoolingLayer):
            lau = l.local_att
            d = {"dnn_kernels": [t(k) for k in lau.dnn.kernels], "dnn_biases": [t(b) for b in lau.dnn.bias],
                 "kernel": t(lau.kernel), "bias": t(lau.bias)}
            acts = []
            for al in lau.dnn.activation_layers:
                if al is not None and al.__class__.__name__ == "Dice":
                    acts.append({"alphas": t(al.alphas), "moving_mean": t(al.moving_mean),
                                 "moving_var": t(al.moving_variance)})
                else:
                    acts.append(None)
            if any(a is not None for a in acts):
                d["act_params"] = acts
            W["lau"] = d
        elif isinstance(l, DNN):
            W["dnn_kernels"] = [t(k) for k in l.kernels]
            W["dnn_biases"] = [t(b) for b in l.bias]
        elif isinstance(l, Linear):
            if l.mode in (1, 2):
                W["linear_kernel"] = t(l.kernel)
        elif isinstance(l, PredictionLayer):
            if l.use_bias:
                W["global_bias"] = t(l.global_bias)
        elif isinstance(l, CIN):
            W["cin_filters"] = [t(f) for f in l.filters]
            W["cin_biases"] = [t(b) for b in l.bias]
        elif isinstance(l, CrossNet):
            W["cross_kernels"] = [t(k) for k in l.kernels]
            W["cross_biases"] = [t(b) for b in l.bias]
        elif isinstance(l, InteractingLayer):
            d = {"query": t(l.W_Query), "key": t(l.W_key), "value": t(l.W_Value)}
            if l.use_res:
                d["res"] = t(l.W_Res)
            W["att"].append(d)
        elif isinstance(l, Dense):
            denses.append(l)
    W["_dense_layers"] = denses
    if denses:
        W["dense_kernel"] = t(denses[0].kernel)
    if len(denses) > 1:
        W["cin_dense_kernel"] = t(denses[1].kernel)
    return W


def flat_params(W):
    """name -> leaf tensor for every oracle weight (for gradient comparison)."""
    out = {}
    for k, v in W.items():
        if k.startswith("_"):
            continue
        if isinstance(v, torch.Tensor):
            out[k] = v
        elif isinstance(v, dict):
            for k2, v2 in v.items():
                if isinstance(v2, torch.Tensor):
                    out["%s/%s" % (k, k2)] = v2
                elif isinstance(v2, list):
                    for i, e in enumerate(v2):
                        if isinstance(e, torch.Tensor):
                            out["%s/%s/%d" % (k, k2, i)] = e
                        elif isinstance(e, dict):
                            for k3, v3 in e.items():
                                if isinstance(v3, torch.Tensor):
                                    out["%s/%s/%d/%s" % (k, k2, i, k3)] = v3
        elif isinstance(v, list):
            for i, e in enumerate(v):
                if isinstance(e, torch.Tensor):
                    out["%s/%d" % (k, i)] = e
                elif isinstance(e, dict):
                    for k2, v2 in e.items():
                        out["%s/%d/%s" % (k, i, k2)] = v2
    return out


def rel_err(a, b):
    a = np.asarray(a, dtype=np.float64).reshape(-1)
    b = np.asarray(b, dtype=np.float64).reshape(-1)
    return float(np.max(np.abs(a - b) / (np.abs(b) + 1e-6)))
