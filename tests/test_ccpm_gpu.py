"""GPU: CCPM's convolution stack kernels and the CCPM builder.

* b2ctr_conv_stack_fwd / _bwd against float64: one conv stage over widths 1 to 9 (wider than the rows too), rows 1 to
  64, E = 1 / 4 / 5 / 32, 1 to 8 channels in and out and every activation; one k-max stage with k = 1, the rows and
  in between; whole CCPM stacks (the defaults at 26 fields, the reference test's configuration at 3 fields, three
  layers) and the bench shape at a reduced batch.  The input is a window of a wider buffer, dx is added to an
  existing gradient and nothing outside the windows changes;
* k-max selections are exact, gradients through them are checked where the float64 margin exceeds the tolerance, and
  equal values send their gradient to the lower rows;
* the backward is bit-identical from run to run; shapes outside the limits raise ValueError naming them;
* a CCPM forward is one conv_stack_fwd launch (no per-layer launch, no copy), a training step one conv_stack_bwd.
Fixtures (with model_golden_checks): the Conv2D / KMaxPooling layer fixtures and the model fixtures' logits and one
SGD step in both GEMM precisions; a graph-replayed CCPM step equals an eager one; every update policy behaves as
for DCN.
"""
import numpy as np
import pytest
import torch

import model_golden_checks as C
import ccpm_family  # noqa: F401  (registers the "ccpm" fixture families)
import ccpm_oracle as CO

pytestmark = pytest.mark.gpu

T = C.gpu_model_tests("ccpm")
test_model_forward_matches_reference = T.forward
test_model_sgd_step_matches_reference_gradients = T.sgd_step
test_layer_fixture = C.gpu_layer_test("ccpm")
test_graph_replayed_step_equals_eager = C.graph_replay_test([
    pytest.param("CCPM", dict(n_dense=0), id="ccpm_defaults"),
    pytest.param("CCPM", dict(n_dense=0, conv_kernel_width=(4, 3, 2), conv_filters=(3, 2, 2)), id="ccpm_three")])

ACTS = (None, "relu", "sigmoid", "tanh")


def _stages(spec, C_in, g, cuda):
    """spec: ('conv', width, filters, act) / ('kmax', k) -> the kernel's stages with random float32 weights."""
    out, c = [], C_in
    for st in spec:
        if st[0] == "conv":
            _, w, f, act = st
            kern = (torch.randn((w, 1, c, f), generator=g, device=cuda) / np.sqrt(w * c)).contiguous()
            bias = 0.1 * torch.randn((f,), generator=g, device=cuda)
            out.append(("conv", w, f, act, kern, bias))
            c = f
        else:
            out.append(st)
    return out


def _ref64(stages, x64):
    h = x64
    for st in stages:
        if st[0] == "conv":
            h = CO.conv2d(h, st[4].double().requires_grad_(True), st[5].double().requires_grad_(True), st[3])
        else:
            h = CO.kmax(h, st[1], 1)
    return h


def _margins(stages, x64):
    """Per (sample, e) column, the smallest relative gap between consecutive sorted values down to the (k+1)-th of
    every k-max stage, in float64."""
    h, m = x64.detach(), None
    for st in stages:
        if st[0] == "conv":
            h = CO.conv2d(h, st[4].double(), st[5].double(), st[3])
        else:
            v, _ = torch.sort(h, dim=1, descending=True)
            top = v[:, :min(st[1] + 1, v.shape[1])]
            if top.shape[1] > 1:
                gap = (top[:, :-1] - top[:, 1:]).abs() / top[:, :-1].abs().clamp_min(1e-30)
                gm = gap.amin(dim=(1, 3))
                m = gm if m is None else torch.minimum(m, gm)
            h = v[:, :st[1]]
    return m


def _check(cuda, spec, B, rows, E, C_in, seed, tol=2e-5):
    """Forward and dx of the stack ``spec`` against float64: output window and dx window of wider buffers, dx added
    to an existing gradient; dx compared on the columns whose k-max margins exceed 1e-4."""
    from deepctr_b200 import kernels as K
    g = torch.Generator(device=cuda).manual_seed(seed)
    stages = _stages(spec, C_in, g, cuda)
    w_in = rows * E * C_in
    k_out, c_out = K.conv_stack_check(rows, C_in, stages)
    w_out = k_out * E * c_out
    xbuf = torch.randn((B, 5 + w_in + 3), generator=g, device=cuda)
    x = xbuf[:, 5:5 + w_in]
    obuf = torch.full((B, 2 + w_out + 6), 7.0, device=cuda)
    K.conv_stack_fwd(stages, x, rows, E, C_in, B, obuf[:, 2:2 + w_out])
    x64 = x.double().reshape(B, rows, E, C_in).requires_grad_(True)
    y64 = _ref64(stages, x64)
    got = obuf[:, 2:2 + w_out].double().reshape(y64.shape)
    assert torch.all(obuf[:, :2] == 7) and torch.all(obuf[:, 2 + w_out:] == 7)
    err = float((got - y64.detach()).abs().max())
    assert err <= tol * max(1.0, float(y64.detach().abs().max())), err
    # backward: dx added to an existing gradient window
    gbuf = torch.randn((B, 1 + w_out + 4), generator=g, device=cuda)
    dout = gbuf[:, 1:1 + w_out]
    dxbuf = torch.randn((B, 3 + w_in + 2), generator=g, device=cuda)
    before = dxbuf.clone()
    want_dw = [st[0] == "conv" for st in stages]
    K.conv_stack_bwd(stages, x, rows, E, C_in, B, dout, dx=dxbuf[:, 3:3 + w_in], dx_accumulate=True,
                     want_dw=want_dw)
    (y64 * dout.double().reshape(y64.shape)).sum().backward()
    assert torch.equal(dxbuf[:, :3], before[:, :3]) and torch.equal(dxbuf[:, 3 + w_in:], before[:, 3 + w_in:])
    dx = (dxbuf[:, 3:3 + w_in] - before[:, 3:3 + w_in]).double().reshape(x64.shape)
    m = _margins(stages, x64)
    ok = torch.ones((B, E), dtype=torch.bool, device=cuda) if m is None else m > 1e-4
    assert float(ok.float().mean()) > 0.9
    gx = x64.grad
    sel = ok[:, None, :, None].expand_as(dx)
    scale = max(1.0, float(gx.abs().max()))
    gerr = float((dx - gx)[sel].abs().max()) if bool(sel.any()) else 0.0
    assert gerr <= 1e-4 * scale, gerr


def _weight_grads64(stages, x64, dout):
    """Per conv stage, the float64 (dkernel, dbias) and the sums of the absolute values of their terms (the scale
    of a float32 sum's rounding)."""
    ws, h = [], x64.detach()
    for st in stages:
        if st[0] == "conv":
            k, b = st[4].double().requires_grad_(True), st[5].double().requires_grad_(True)
            z = CO.conv2d(h, k, b, None)
            z.retain_grad()
            ws.append((k, b, h, z))
            h = CO._ACT[st[3]](z)
        else:
            h = CO.kmax(h, st[1], 1)
    (h * dout.double().reshape(h.shape)).sum().backward()
    out = []
    for k, b, hin, z in ws:
        w = k.shape[0]
        pb = (w - 1) // 2
        hp = torch.nn.functional.pad(hin.abs().permute(0, 3, 1, 2), (0, 0, pb, w - 1 - pb))
        dz = z.grad.abs().permute(0, 3, 1, 2)
        kabs = torch.nn.grad.conv2d_weight(hp, (k.shape[3], k.shape[2], w, 1), dz).permute(2, 3, 1, 0)
        out.append(((k.grad, kabs), (b.grad, dz.sum(dim=(0, 2, 3)))))
    return out


def _check_dw(cuda, spec, B, rows, E, C_in, seed):
    """The weight gradients against float64 (inputs and weights as _check draws them), within 2e-5 of the sum of
    the absolute values of their terms."""
    from deepctr_b200 import kernels as K
    g = torch.Generator(device=cuda).manual_seed(seed)
    stages = _stages(spec, C_in, g, cuda)
    w_in = rows * E * C_in
    k_out, c_out = K.conv_stack_check(rows, C_in, stages)
    w_out = k_out * E * c_out
    x = torch.randn((B, 5 + w_in + 3), generator=g, device=cuda)[:, 5:5 + w_in]
    dout = torch.randn((B, w_out), generator=g, device=cuda)
    dws = K.conv_stack_bwd(stages, x, rows, E, C_in, B, dout, want_dw=[st[0] == "conv" for st in stages])
    ref = _weight_grads64(stages, x.double().reshape(B, rows, E, C_in), dout)
    for (dk, db), pairs in zip([d for d in dws if d is not None], ref):
        for got, (want, mag) in zip((dk, db), pairs):
            err = (got.double() - want).abs()
            bound = 2e-5 * mag + 1e-6 * max(1.0, float(want.abs().max()))
            assert bool(torch.all(err <= bound)), float((err / bound).max())


ONE_CONV = [(1, 1, 1), (4, 1, 4), (5, 4, 4), (32, 4, 8), (4, 8, 1), (1, 8, 8)]     # (E, C_in, C_out)


@pytest.mark.parametrize("width", [1, 2, 5, 6, 7, 9])
@pytest.mark.parametrize("rows", [1, 2, 3, 26, 64])
def test_one_conv_stage_matches_float64(cuda, width, rows):
    from deepctr_b200 import kernels as K
    for i, (E, ci, co) in enumerate(ONE_CONV):
        try:
            K.conv_stack_check(rows, ci, [("conv", width, co)])
        except ValueError:
            continue
        act = ACTS[(i + width + rows) % 4]
        spec = [("conv", width, co, act)]
        _check(cuda, spec, 37, rows, E, ci, 100 * width + rows + i)
        _check_dw(cuda, spec, 37, rows, E, ci, 100 * width + rows + i)


@pytest.mark.parametrize("act", ACTS)
def test_every_activation_on_the_default_first_layer(cuda, act):
    _check(cuda, [("conv", 6, 4, act)], 53, 26, 4, 1, 7)
    _check_dw(cuda, [("conv", 6, 4, act)], 53, 26, 4, 1, 7)


@pytest.mark.parametrize("k", [1, 2, 13, 26])
def test_one_kmax_stage_selects_exactly(cuda, k):
    from deepctr_b200 import kernels as K
    B, rows, E, Cc = 41, 26, 5, 3
    g = torch.Generator(device=cuda).manual_seed(k)
    x = torch.randn((B, 2 + rows * E * Cc), generator=g, device=cuda)[:, 2:]
    out = torch.empty((B, k * E * Cc), device=cuda)
    K.conv_stack_fwd([("kmax", k)], x, rows, E, Cc, B, out)
    want = CO.kmax(x.double().reshape(B, rows, E, Cc), k, 1).float()
    assert torch.equal(out.reshape(want.shape), want)
    _check(cuda, [("kmax", k)], B, rows, E, Cc, k)


def test_equal_values_send_the_gradient_to_the_lower_rows(cuda):
    from deepctr_b200 import kernels as K
    B, rows, E = 8, 5, 3
    v = torch.randn((B, 1, E, 1), device=cuda)
    x = v.expand(B, rows, E, 1).contiguous().reshape(B, -1)
    out = torch.empty((B, 3 * E), device=cuda)
    K.conv_stack_fwd([("kmax", 3)], x, rows, E, 1, B, out)
    assert torch.equal(out.reshape(B, 3, E), v.reshape(B, 1, E).expand(B, 3, E))
    dout = torch.randn((B, 3 * E), device=cuda)
    dx = torch.empty_like(x)
    K.conv_stack_bwd([("kmax", 3)], x, rows, E, 1, B, dout, dx=dx)
    dx = dx.reshape(B, rows, E)
    assert torch.equal(dx[:, :3], dout.reshape(B, 3, E)) and torch.all(dx[:, 3:] == 0)


STACKS = {
    "defaults_26": ([("conv", 6, 4, "tanh"), ("kmax", 13), ("conv", 5, 4, "tanh"), ("kmax", 3)], 26),
    "reference_test_3": ([("conv", 3, 2, "tanh"), ("kmax", 3), ("conv", 2, 1, "tanh"), ("kmax", 3)], 3),
    "three_layers_10": ([("conv", 4, 3, "tanh"), ("kmax", 8), ("conv", 3, 2, "tanh"), ("kmax", 3),
                         ("conv", 2, 2, "tanh"), ("kmax", 3)], 10),
}


@pytest.mark.parametrize("stack", sorted(STACKS))
@pytest.mark.parametrize("E", [1, 4, 5, 32])
def test_ccpm_stacks_match_float64(cuda, stack, E):
    spec, rows = STACKS[stack]
    _check(cuda, spec, 29, rows, E, 1, E)
    _check_dw(cuda, spec, 29, rows, E, 1, E)


def test_bench_shape(cuda):
    spec, rows = STACKS["defaults_26"]
    _check(cuda, spec, 8192, rows, 32, 1, 3)
    _check_dw(cuda, spec, 8192, rows, 32, 1, 3)


def test_backward_is_deterministic(cuda):
    from deepctr_b200 import kernels as K
    spec, rows = STACKS["defaults_26"]
    g = torch.Generator(device=cuda).manual_seed(11)
    stages = _stages(spec, 1, g, cuda)
    B, E = 30000, 4
    x = torch.randn((B, rows * E), generator=g, device=cuda)
    dout = torch.randn((B, 3 * E * 4), generator=g, device=cuda)
    runs = []
    for _ in range(2):
        dx = torch.empty_like(x)
        dws = K.conv_stack_bwd(stages, x, rows, E, 1, B, dout, dx=dx, want_dw=[True, False, True, False])
        runs.append([dx] + [t for d in dws if d is not None for t in d])
    for a, b in zip(*runs):
        assert torch.equal(a, b)


@pytest.mark.parametrize("rows,C_in,spec,limit", [
    (65, 1, [("conv", 3, 2, "tanh")], "rows"), (26, 1, [("conv", 33, 2, "tanh")], "width"),
    (26, 1, [("conv", 3, 17, "tanh")], "filters"), (64, 8, [("conv", 3, 8, "tanh")], "shared memory"),
    (26, 1, [("kmax", 27)], "k")])
def test_shapes_outside_the_limits_raise(cuda, rows, C_in, spec, limit):
    from deepctr_b200 import kernels as K
    g = torch.Generator(device=cuda).manual_seed(0)
    stages = _stages(spec, C_in, g, cuda)
    x = torch.randn((4, rows * 2 * C_in), device=cuda)
    out = torch.empty((4, 64 * 2 * 17), device=cuda)
    with pytest.raises(ValueError, match=limit):
        K.conv_stack_fwd(stages, x, rows, 2, C_in, 4, out)


def _ccpm_model(n=512, F=6, V=40, E=4, **kw):
    from deepctr_b200 import engine as E_, models as M
    from deepctr_b200.feature_column import SparseFeat
    rng = np.random.RandomState(3)
    cols = [SparseFeat("C%d" % i, V, E) for i in range(F)]
    x = {"C%d" % i: rng.randint(0, V, size=n).astype(np.int32) for i in range(F)}
    y = (rng.rand(n) < 0.3).astype(np.float32)
    E_.clear_session()
    return M.CCPM(cols, cols, l2_reg_embedding=0, l2_reg_linear=0, **kw), x, y


def test_one_launch_forward_and_backward(cuda):
    from deepctr_b200 import kernels as K
    from deepctr_b200.engine import SGD
    model, x, y = _ccpm_model(conv_kernel_width=(4, 3, 2), conv_filters=(3, 2, 2))
    model.compile(SGD(0.01), "binary_crossentropy", step_graph="off")
    model.predict(x, batch_size=512)
    K.PROFILE = {}
    try:
        model.predict(x, batch_size=512)
        fwd = {k: len(v) for k, v in K.PROFILE.items()}
        K.PROFILE = {}
        model.train_on_batch(x, y)
        step = {k: len(v) for k, v in K.PROFILE.items()}
    finally:
        K.PROFILE = None
    assert fwd.get("conv_stack_fwd") == 1 and "conv_stack_bwd" not in fwd, fwd
    assert "copy2d" not in fwd and "ewise" not in fwd, fwd
    assert step.get("conv_stack_fwd") == 1 and step.get("conv_stack_bwd") == 1, step


@pytest.mark.parametrize("mode", ["dense", "sparse"])
@pytest.mark.parametrize("opt", ["sgd", "adam", "adagrad"])
def test_training_steps_run_with_each_update_policy(cuda, mode, opt):
    """'dense' and 'sparse' updates with SGD, Adam and Adagrad, as for DCN."""
    from deepctr_b200 import engine as E_
    from deepctr_b200 import models as M
    from deepctr_b200.feature_column import SparseFeat
    rng = np.random.RandomState(5)
    cols = [SparseFeat("C%d" % i, 40, 4) for i in range(5)]
    x = {"C%d" % i: rng.randint(0, 40, size=256).astype(np.int32) for i in range(5)}
    y = (rng.rand(256) < 0.3).astype(np.float32)
    results = {}
    for builder in ("DCN", "CCPM"):
        E_.clear_session()
        model = getattr(M, builder)(cols, cols, l2_reg_embedding=0, l2_reg_linear=0)
        optimizer = {"sgd": E_.SGD(0.05), "adam": E_.Adam(0.01), "adagrad": E_.Adagrad(0.05)}[opt]
        try:
            model.compile(optimizer, "binary_crossentropy", embedding_update=mode)
            losses = [model.train_on_batch(x, y) for _ in range(3)]
            results[builder] = ("ok", bool(np.all(np.isfinite(losses))))
        except ValueError as e:
            results[builder] = ("error", str(e).split(":")[0])
    assert results["CCPM"] == results["DCN"], results
