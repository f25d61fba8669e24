"""GPU parity AT THE BASELINE.json SHAPES (vocabularies reduced so that the CPU oracle finishes in seconds;
everything that selects kernels - F, E, batch, K of the first GEMM, CIN sizes, T, attention sizes - is the
bench configuration's).  Every step: the loss against the oracle evaluated on the model's CURRENT weights
(logits within 1e-4, north_star); on the graph-replayed step also every weight update against the oracle's
autograd gradient.

  C2  DeepFM   F=26 E=32 B=65536 (K=845 first GEMM, the many-tile persistent wgmma path, graph replay)
  C3  xDeepFM  F=26 E=16 CIN (128,128) split_half relu, B=4096
  C4  DIN      T=50 E=64 att (80,40), B=2048: sigmoid (training step) and dice (inference statistics)
"""
import numpy as np
import pytest
import torch

import b2_helpers as H
import bench as BN
from oracle import models as OM
from oracle import ops as O

pytestmark = pytest.mark.gpu


def _setup(cfg, act=None, std=0.05):
    from deepctr_b200 import engine as E, ops
    ops.set_gemm_precision("bf16x3")             # what bench.py measures
    E.clear_session()
    rng = np.random.RandomState(7)
    model = BN.build_model(cfg, act=act)
    H.randomize_weights(model, rng, std=std)
    cols = BN.feature_columns(cfg)
    data = [(BN.user_inputs(x), y) for x, y in BN.synth_batches(cfg, 3, 0, "uniform")]
    return model, cols, data


def _oracle(cfg, cols, x, W, act="sigmoid", training=False):
    if cfg["kind"] == "deepfm":
        return OM.deepfm(x, cols, cols, W)
    if cfg["kind"] == "xdeepfm":
        return OM.xdeepfm(x, cols, cols, W, cin_layer_size=cfg["cin"])
    return OM.din(x, cols, ["item_id"], W, att_activation=act, training=training)


def _check_steps(cfg, model, cols, data, lr, nsteps, act="sigmoid", check_update_at=None, upd_tol=3e-3):
    """train_on_batch over the batches (the staging ring turns step >= 3 into graph replays)."""
    for step in range(nsteps):
        x, y = data[step % len(data)]
        W = H.oracle_weights(model, requires_grad=step == check_update_at)
        logit, pred = _oracle(cfg, cols, x, W, act=act, training=True)
        want = O.binary_crossentropy(y, pred)
        if step == check_update_at:
            want.backward()
        got = model.train_on_batch(x, y)
        assert abs(got - float(want.detach())) < 1e-4 * max(1.0, abs(float(want.detach()))), (step, got, float(want.detach()))
        if step == check_update_at:
            new, old = H.flat_params(H.oracle_weights(model)), H.flat_params(W)
            for name, p in old.items():
                if p.grad is None:
                    continue
                upd = lr * p.grad.numpy()
                w0 = p.detach().numpy()
                # w += delta rounds to an ulp of |w| however it is computed (one add on the CPU, one atomic add
                # per duplicate id on the GPU): at these batch sizes an update is only ~100 ulps of its weight
                ulp = 4.0 * np.finfo(np.float32).eps * float(np.abs(w0).max())
                err = (np.abs(new[name].numpy() - (w0 - upd)).max() - ulp) / (np.abs(upd).max() + 1e-12)
                # a bias gradient is a column sum over B (x D) rows of relu-masked terms: pre-activations within the
                # split-bf16 error of zero flip their mask against the fp32 oracle, and the sum cancels to a small
                # total, so a handful of flipped terms is a visible fraction of it
                tol = 10 * upd_tol if "bias" in name else upd_tol
                assert err < tol, "step %d weight %s: update mismatch %.3e (relative to max update)" % (step, name, err)


def _logits(model, x):
    from deepctr_b200 import engine as E
    model._materialize()
    feed = model._feed(x)
    logit_t, head = model._head()
    vals = model._run(feed, False, upto=head)
    return E.contiguous(vals[id(logit_t)]).reshape(-1, 1).cpu().numpy()


def _check_logits(cfg, model, cols, x, n, act="sigmoid"):
    """fp32 logits within 1e-4 relative (north_star); normwise floor 1e-4 * max|logit| for the split-bf16 GEMMs."""
    xs = {k: v[:n] for k, v in x.items()}
    W = H.oracle_weights(model)
    logit, pred = _oracle(cfg, cols, xs, W, act=act, training=False)
    want = logit.numpy().reshape(-1, 1)
    got = _logits(model, xs)
    np.testing.assert_allclose(got, want, rtol=1e-4, atol=1e-4 * float(np.abs(want).max()))
    np.testing.assert_allclose(model.predict(xs, batch_size=n), pred.numpy().reshape(-1, 1), rtol=1e-4, atol=2e-5)


def test_c2_shaped_deepfm_step(cuda):
    from deepctr_b200.engine import SGD
    cfg = dict(BN.CONFIGS["c2"], vocab=100000)
    model, cols, data = _setup(cfg)
    lr = 0.05
    model.compile(SGD(lr), "binary_crossentropy", embedding_update="sparse")
    _check_steps(cfg, model, cols, data, lr, 5, check_update_at=3)
    assert model._step_graphs and model.replayed_launches > 0           # steps 2.. ran as graph replays
    p = model.planner
    assert p.fast and p.fm_hint is not None and p.lin_hint and p.tail_hint is not None
    _check_logits(cfg, model, cols, data[0][0], 4096)


def test_c3_shaped_xdeepfm_step(cuda):
    from deepctr_b200.engine import SGD
    cfg = dict(BN.CONFIGS["c3"], vocab=10000, batch=4096)
    model, cols, data = _setup(cfg)
    lr = 0.05
    model.compile(SGD(lr), "binary_crossentropy", embedding_update="sparse")
    _check_steps(cfg, model, cols, data, lr, 4, check_update_at=3)
    _check_logits(cfg, model, cols, data[0][0], 2048)


@pytest.mark.parametrize("act", ["sigmoid", "dice"])
def test_c4_shaped_din(cuda, act):
    from deepctr_b200.engine import SGD
    cfg = dict(BN.CONFIGS["c4"], vocab=5001, batch=2048)
    model, cols, data = _setup(cfg, act=act, std=0.1)
    lr = 0.05
    model.compile(SGD(lr), "binary_crossentropy", embedding_update="sparse")
    _check_logits(cfg, model, cols, data[0][0], 2048, act=act)          # dice: moving (inference) statistics
    if act == "sigmoid":
        _check_steps(cfg, model, cols, data, lr, 4, act=act, check_update_at=3)
        _check_logits(cfg, model, cols, data[1][0], 1024, act=act)
