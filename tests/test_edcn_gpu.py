"""GPU: EDCN's bridge-and-regulate kernels and the EDCN builder.

* b2ctr_regulate_fwd / _bwd against float64 for every mode (copy / add / hadamard / attention) and output set
  ({u}, {y0}, {y0, y1}, {u, y0, y1}), over F = 3 / 26 / 64 and E = 4 / 5 / 16 (E = 5 takes the scalar path) with
  tau = 1 and 0.5, every operand and output a window of a wider buffer and dx added to an existing gradient; and at
  the bench shape (26 fields, E = 16) with a reduced batch;
* the backward is bit-identical from run to run;
* shapes outside the limits raise ValueError naming them;
* a forward with cross_num = 3 issues cross_num + 1 regulate launches (cross_num for 'concatenation') and no
  separate bridge, reshape or gate kernel: the inner bridge outputs are never written.
Model fixtures (with model_golden_checks): logits and one SGD step in both GEMM precisions; a graph-replayed EDCN step
equals an eager one for a vector and a matrix configuration.
"""
import numpy as np
import pytest
import torch

import model_golden_checks as C
import edcn_family  # noqa: F401  (registers the "edcn" fixture family)

pytestmark = pytest.mark.gpu

T = C.gpu_model_tests("edcn")
test_model_forward_matches_reference = T.forward
test_model_sgd_step_matches_reference_gradients = T.sgd_step
test_graph_replayed_step_equals_eager = C.graph_replay_test([
    pytest.param("EDCN", dict(n_dense=0, bridge_type="hadamard_product"), id="edcn_vector_hadamard"),
    pytest.param("EDCN", dict(n_dense=0, cross_parameterization="matrix", bridge_type="attention_pooling"),
                 id="edcn_matrix_attention")])

MODES = ("copy", "add", "hadamard", "attention")
OUTPUTS = {"u": (True, 0), "y0": (False, 1), "y0y1": (False, 2), "uy0y1": (True, 2)}


def _wide(g, B, d, cuda, lo=4, hi=8):
    """A [B, d] window at column ``lo`` of a [B, lo + d + hi] buffer of random values."""
    return torch.randn((B, lo + d + hi), generator=g, device=cuda)[:, lo:lo + d]


def _v64(mode, x, h, ax, ah):
    x = x.double().cpu()
    if mode == "copy":
        return x
    h = h.double().cpu()
    if mode == "add":
        return x + h
    if mode == "hadamard":
        return x * h
    return ax.double().cpu() * x + ah.double().cpu() * h


def _check(cuda, mode, outputs, B, F, E, tau, seed):
    from deepctr_b200 import kernels as K
    g = torch.Generator(device=cuda).manual_seed(seed)
    d = F * E
    x, h = _wide(g, B, d, cuda), _wide(g, B, d, cuda, lo=8, hi=4)
    ax = torch.softmax(_wide(g, B, d, cuda), -1) if mode == "attention" else None
    ah = torch.softmax(_wide(g, B, d, cuda, lo=12), -1) if mode == "attention" else None
    if mode == "copy":
        h = None
    want_u, ngates = OUTPUTS[outputs]
    gw = [torch.randn((1, F, 1), generator=g, device=cuda) for _ in range(ngates)]
    gates = [(w.reshape(-1), 1.0 / tau) for w in gw]
    bufs = [torch.full((B, d + 12), 7.0, device=cuda) for _ in range(int(want_u) + ngates)]
    wins = [(b_, 4) for b_ in bufs]
    u = wins[0] if want_u else None
    ys = wins[1:] if want_u else wins
    K.regulate_fwd(mode, F, E, B, x, h, ax, ah, gates, u=u, y0=ys[0] if ngates > 0 else None,
                   y1=ys[1] if ngates > 1 else None)
    v = _v64(mode, x, h, ax, ah)
    gate64 = [torch.softmax(w.double().cpu().reshape(F) / tau, 0) for w in gw]
    want = ([v] if want_u else []) + [(v.reshape(B, F, E) * gk[None, :, None]).reshape(B, d) for gk in gate64]
    for buf, w in zip(bufs, want):
        got = buf.cpu()
        np.testing.assert_allclose(got[:, 4:4 + d].double().numpy(), w.numpy(), rtol=1e-5, atol=1e-6)
        assert bool((got[:, :4] == 7).all()) and bool((got[:, 4 + d:] == 7).all())      # nothing outside the window
    # ---- backward: incoming gradients as windows, dx added to an existing gradient ----
    grads = [torch.randn((B, d + 8), generator=g, device=cuda) for _ in bufs]
    gwin = [(t, 4) for t in grads]
    du = gwin[0] if want_u else None
    dys = gwin[1:] if want_u else gwin
    dxbuf = torch.randn((B, d + 8), generator=g, device=cuda)
    dx0 = dxbuf.clone()

    def run(dxb):
        return K.regulate_bwd(mode, F, E, B, x, h, ax, ah, gates, du=du, dy0=dys[0] if ngates > 0 else None,
                              dy1=dys[1] if ngates > 1 else None, dx=dxb[:, 4:4 + d], dx_accumulate=True,
                              want_dh=h is not None, want_dax=ax is not None, want_dah=ah is not None,
                              want_dg=[True] * ngates + [False] * (2 - ngates))
    _, dh, dax, dah, dg0, dg1 = run(dxbuf)
    g64 = [t[:, 4:4 + d].double().cpu() for t in grads]
    gu = g64[0] if want_u else torch.zeros((B, d), dtype=torch.float64)
    gy = g64[1:] if want_u else g64
    dv = gu.clone()
    for gk, dy in zip(gate64, gy):
        dv += (dy.reshape(B, F, E) * gk[None, :, None]).reshape(B, d)
    xx = x.double().cpu()
    dx_want = {"copy": dv, "add": dv, "hadamard": dv * (h.double().cpu() if h is not None else 0),
               "attention": dv * (ax.double().cpu() if ax is not None else 0)}[mode]
    got_dx = dxbuf.cpu().double()
    np.testing.assert_allclose(got_dx[:, 4:4 + d].numpy(), (dx0.cpu().double()[:, 4:4 + d] + dx_want).numpy(),
                               rtol=1e-5, atol=1e-5)
    assert torch.equal(dxbuf[:, :4], dx0[:, :4]) and torch.equal(dxbuf[:, 4 + d:], dx0[:, 4 + d:])
    if mode == "add":
        np.testing.assert_allclose(dh.cpu().double().numpy(), dv.numpy(), rtol=1e-5, atol=1e-6)
    elif mode == "hadamard":
        np.testing.assert_allclose(dh.cpu().double().numpy(), (dv * xx).numpy(), rtol=1e-5, atol=1e-6)
    elif mode == "attention":
        np.testing.assert_allclose(dh.cpu().double().numpy(), (dv * ah.double().cpu()).numpy(), rtol=1e-5,
                                   atol=1e-6)
        np.testing.assert_allclose(dax.cpu().double().numpy(), (dv * xx).numpy(), rtol=1e-5, atol=1e-6)
        np.testing.assert_allclose(dah.cpu().double().numpy(), (dv * h.double().cpu()).numpy(), rtol=1e-5,
                                   atol=1e-6)
    for k, (gk, dy, dg) in enumerate(zip(gate64, gy, (dg0, dg1))):
        s = (v * dy).reshape(B, F, E).sum(dim=(0, 2))
        want_dg = (gk * (s - (gk * s).sum())) / tau
        scale = float(np.abs(want_dg.numpy()).max()) + float(s.abs().max()) * 1e-6
        np.testing.assert_allclose(dg.cpu().double().numpy(), want_dg.numpy(), rtol=1e-4, atol=1e-5 * scale,
                                   err_msg="dg%d" % k)


@pytest.mark.parametrize("outputs", list(OUTPUTS))
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("F,E,tau", [(3, 4, 1.0), (3, 5, 0.5), (3, 16, 1.0), (26, 4, 0.5), (26, 5, 1.0),
                                     (26, 16, 0.5), (64, 4, 1.0), (64, 5, 0.5), (64, 16, 1.0)])
def test_regulate_matches_float64(cuda, mode, outputs, F, E, tau):
    _check(cuda, mode, outputs, 257, F, E, tau, seed=F * 100 + E)


@pytest.mark.parametrize("mode", MODES)
def test_regulate_bench_shape(cuda, mode):
    """26 fields x E = 16 (d = 416), u and both gates, B = 8192."""
    _check(cuda, mode, "uy0y1", 8192, 26, 16, 1.0, seed=5)


@pytest.mark.parametrize("E", [16, 5])
def test_regulate_backward_is_deterministic(cuda, E):
    from deepctr_b200 import kernels as K
    g = torch.Generator(device=cuda).manual_seed(11)
    B, F = 30000, 26
    d = F * E
    x, h, ax, ah = (torch.randn((B, d), generator=g, device=cuda) for _ in range(4))
    gates = [(torch.randn((F,), generator=g, device=cuda), 2.0) for _ in range(2)]
    du, dy0, dy1 = (torch.randn((B, d), generator=g, device=cuda) for _ in range(3))
    runs = []
    for _ in range(2):
        runs.append(K.regulate_bwd("attention", F, E, B, x, h, ax, ah, gates, du=(du, 0), dy0=(dy0, 0),
                                   dy1=(dy1, 0), want_dh=True, want_dax=True, want_dah=True, want_dg=(True, True)))
    for a, b in zip(*runs):
        assert torch.equal(a, b)


@pytest.mark.parametrize("F,E,what", [(1025, 4, "field count <= 1024"), (4, 257, "embedding_size <= 256")])
def test_shapes_outside_the_limits_raise(cuda, F, E, what):
    from deepctr_b200 import kernels as K
    x = torch.zeros((2, F * E), device=cuda)
    g = torch.zeros((F,), device=cuda)
    y = torch.empty((2, F * E), device=cuda)
    with pytest.raises(ValueError, match=what):
        K.regulate_fwd("copy", F, E, 2, x, gates=[(g, 1.0)], y0=(y, 0))
    with pytest.raises(ValueError, match=what):
        K.regulate_bwd("copy", F, E, 2, x, gates=[(g, 1.0)], dy0=(y, 0))


def _edcn_model(bridge_type, cross_num, n=512, F=6, V=40, E=4):
    from deepctr_b200 import engine as E_, models as M
    from deepctr_b200.feature_column import SparseFeat
    rng = np.random.RandomState(3)
    cols = [SparseFeat("C%d" % i, V, E) for i in range(F)]
    x = {"C%d" % i: rng.randint(0, V, size=n).astype(np.int32) for i in range(F)}
    E_.clear_session()
    return M.EDCN(cols, cols, cross_num=cross_num, bridge_type=bridge_type), x


@pytest.mark.parametrize("bridge_type", ["pointwise_addition", "hadamard_product", "concatenation",
                                         "attention_pooling"])
def test_inner_bridge_outputs_are_not_materialised(cuda, bridge_type):
    """cross_num = 3: one launch for layer 0's gates, one per inner boundary and, unless the bridge is
    'concatenation' (Dense on the GEMM), one for the last bridge; no elementwise kernel, and no copy besides the
    concatenations'."""
    from deepctr_b200 import kernels as K
    model, x = _edcn_model(bridge_type, 3)
    model.predict(x, batch_size=512)                   # warm up: weights, staging buffers
    K.PROFILE = {}
    try:
        model.predict(x, batch_size=512)
        launched = {k: len(v) for k, v in K.PROFILE.items()}
    finally:
        K.PROFILE = None
    concat = bridge_type == "concatenation"
    assert launched.get("regulate_fwd", 0) == (3 if concat else 4), launched
    assert "ewise" not in launched, launched
    # the final Concatenate copies its three inputs; a 'concatenation' bridge copies its two inputs
    assert launched.get("copy2d", 0) == 3 + (6 if concat else 0), launched


@pytest.mark.parametrize("mode", ["dense", "sparse"])
@pytest.mark.parametrize("opt", ["sgd", "adam", "adagrad"])
def test_training_steps_run_with_each_update_policy(cuda, mode, opt):
    """'dense' and 'sparse' updates with SGD, Adam and Adagrad, as for DCN (Adam keeps dense state, so 'sparse'
    Adam is rejected there as it is here)."""
    from deepctr_b200 import engine as E_
    from deepctr_b200 import models as M
    from deepctr_b200.feature_column import SparseFeat
    rng = np.random.RandomState(5)
    cols = [SparseFeat("C%d" % i, 40, 4) for i in range(5)]
    x = {"C%d" % i: rng.randint(0, 40, size=256).astype(np.int32) for i in range(5)}
    y = (rng.rand(256) < 0.3).astype(np.float32)
    results = {}
    for builder in ("DCN", "EDCN"):
        E_.clear_session()
        kw = dict(l2_reg_embedding=0, l2_reg_linear=0)
        model = getattr(M, builder)(cols, cols, **kw)
        optimizer = {"sgd": E_.SGD(0.05), "adam": E_.Adam(0.01), "adagrad": E_.Adagrad(0.05)}[opt]
        try:
            model.compile(optimizer, "binary_crossentropy", embedding_update=mode)
            losses = [model.train_on_batch(x, y) for _ in range(3)]
            results[builder] = ("ok", bool(np.all(np.isfinite(losses))))
        except ValueError as e:
            results[builder] = ("error", str(e).split(":")[0])
    assert results["EDCN"] == results["DCN"], results
