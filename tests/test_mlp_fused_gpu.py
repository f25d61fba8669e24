"""GPU: the fused relu tower (b2ctr_mlp_relu_fwd / _bwd and ops.mlp) against float64 and against the per-layer path.

- exact-valued operands (integers times powers of two): the weights are bf16-exact (their lo planes are zero) and
  every activation and gradient stays below 2^16 grid units, so the split-bf16 product is exact; every partial sum
  stays below 2^24 units, so the kernels must equal float64 bit for bit, and every plane byte must equal
  split_planes of the exact tensor.  The weights have at most four nonzeros per row and per column, which bounds
  both directions' sums.
- random operands: ops.mlp and the per-layer ops.dense loop, each against float64 within the bound
  tests/test_dense_tower_gpu.py derives (2^-15 sum|a||b| for the split-bf16 product plus the fp32 accumulation).
"""
import zlib

import pytest
import torch

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
LIMIT = 2.0 ** 24
TOWERS = [(256, 128, 64), (128, 128, 64), (256, 128), (128, 64)]
BATCHES = [65536, 1, 63, 64, 127, 129, 255, 257, 65535]


def _mods():
    from deepctr_b200 import _lib as L, kernels as K, ops, engine as E
    return L, K, ops, E


@pytest.fixture
def gen(cuda, request):
    g = torch.Generator(device=cuda)
    g.manual_seed(zlib.crc32(request.node.name.encode()))
    return g


def _ints(gen, shape, lo, hi, scale):
    return torch.randint(lo, hi + 1, shape, generator=gen, device=gen.device).float() * scale


def _sparse_sign(gen, k, n, scale):
    """[k, n] with entries +-scale, at most four nonzeros per row and per column"""
    w = torch.zeros((k, n), device=gen.device)
    for _ in range(4):
        rows = torch.randperm(max(k, n), generator=gen, device=gen.device)
        r, c = rows[:n] % k, torch.arange(n, device=gen.device)
        keep = rows[:n] < k
        sign = torch.randint(0, 2, (n,), generator=gen, device=gen.device).float() * 2 - 1
        w[r[keep], c[keep]] = sign[keep] * scale
    return w


def _equal(got, ref, what):
    want = ref.float()
    assert bool((want.double() == ref).all()), what + ": reference not representable in fp32 (test bug)"
    if not torch.equal(got, want):
        d = (got.double() - ref).abs()
        raise AssertionError("%s: %d elements differ, max |diff| %.3e" % (what, int((d > 0).sum()), float(d.max())))


def _used(planes, rows, cols):
    """both planes, pad rows and columns included; the buffer's trailing slack is written by no kernel"""
    return planes[:(rows + 255) // 256 * 256 * (64 if cols <= 64 else (cols + 127) // 128 * 128) * 4]


def _bytes_equal(K, got, exact, what):
    want = K.split_planes(exact.float().contiguous())
    assert got.shape == want.shape, what
    got, want = _used(got, *exact.shape), _used(want, *exact.shape)
    if not torch.equal(got, want):
        raise AssertionError("%s: %d of %d plane bytes differ" % (what, int((got != want).sum()), got.numel()))


def _exact_tower(gen, B, widths, zero_rows=True):
    y0 = _ints(gen, (B, widths[0]), 0, 2047, 2.0 ** -5)             # 11 significant bits: the lo plane is used
    y0[::5] *= (y0[::5] >= 2.0 ** -5 * 1024).float()               # exact zeros in y0 (layer 0's relu)
    if zero_rows:
        y0[3::7] = 0.0                                              # these rows reach layer 1 as relu(b)
    ws = [_sparse_sign(gen, widths[i - 1], widths[i], 2.0 ** -3) for i in range(1, len(widths))]
    bs = [_ints(gen, (n,), -64, 64, 2.0 ** -8) for n in widths[1:]]
    for b in bs:
        b[::3] = 0.0                                                # relu(0 + 0) = 0: the mask at exactly 0
    dy = torch.zeros((B, widths[-1]), device=gen.device)
    sel = torch.arange(B, device=gen.device)
    sel = sel[(sel % 128 == 0) | (sel % 128 == 127) | (sel == B - 1)]
    dy[sel] = _ints(gen, (sel.numel(), widths[-1]), -200, 200, 2.0 ** -6)
    return y0, ws, bs, dy


def _reference(y0, ws, bs, dy):
    """float64 forward activations, relu masks, dz of every layer (dz_0 first) and the bias gradients"""
    hs = [y0.double()]
    for w, b in zip(ws, bs):
        hs.append(torch.relu(hs[-1] @ w.double() + b.double()))
    g = dy.double()
    dzs = [None] * len(hs)
    for i in reversed(range(len(hs))):
        dzs[i] = g * (hs[i] > 0).double()
        if i > 0:
            g = dzs[i] @ ws[i - 1].double().t()
    return hs, dzs


@pytest.mark.parametrize("widths", TOWERS, ids=["-".join(map(str, w)) for w in TOWERS])
@pytest.mark.parametrize("B", BATCHES)
def test_mlp_relu_kernels_exact(cuda, gen, B, widths):
    """y_{L-1}, every db_i and every plane buffer (pad rows and columns included) equal float64 / split_planes of
    the exact tensors, and a second run writes the same bytes."""
    L, K, ops, E = _mods()
    y0, ws, bs, dy = _exact_tower(gen, B, widths)
    hs, dzs = _reference(y0, ws, bs, dy)
    for h in hs:
        assert float(h.abs().max()) < 2.0 ** 16 * 2.0 ** -8          # split exactly into hi + lo
    for dz in dzs:
        assert float(dz.abs().sum(0).max()) < LIMIT * 2.0 ** -12     # every column sum exact in fp32
        assert float(dz.abs().max()) < 2.0 ** 16 * 2.0 ** -9
    planes, y = K.mlp_relu_fwd(y0, ws, bs)
    _equal(y, hs[-1], "y_last")
    assert len(planes) == len(widths) - 1
    for i, p in enumerate(planes):
        _bytes_equal(K, p, hs[i], "planes of y_%d" % i)
    dzp, db = K.mlp_relu_bwd(dy, y, y0, planes, ws)
    for i in range(len(widths)):
        _bytes_equal(K, dzp[i], dzs[i], "planes of dz_%d" % i)
        _equal(db[i], dzs[i].sum(0), "db_%d" % i)
    # determinism: bit-identical second run
    planes2, y2 = K.mlp_relu_fwd(y0, ws, bs)
    dzp2, db2 = K.mlp_relu_bwd(dy, y2, y0, planes2, ws)
    assert torch.equal(y, y2)
    for i, (a, b) in enumerate(zip(planes, planes2)):
        assert torch.equal(_used(a, B, widths[i]), _used(b, B, widths[i]))
    for i, (a, b) in enumerate(zip(dzp, dzp2)):
        assert torch.equal(_used(a, B, widths[i]), _used(b, B, widths[i]))
    assert all(torch.equal(a, b) for a, b in zip(db, db2))


def test_mlp_relu_rejects_unsupported(cuda):
    L, K, ops, E = _mods()
    y0 = torch.zeros((256, 256), device=cuda)
    ws = [torch.zeros((256, 96), device=cuda)]
    bs = [torch.zeros((96,), device=cuda)]
    with pytest.raises(ValueError):
        K.mlp_relu_fwd(y0, ws, bs)


def _run_dnn(x_data, widths, kernels, biases, gy, fused):
    """forward + backward of a relu DNN tower through ops.mlp (fused) or the per-layer ops.dense loop"""
    L, K, ops, E = _mods()
    x = E.Var(x_data.clone(), requires_grad=True)
    Ws = [E.Var(w.clone(), requires_grad=True) for w in kernels]
    bs = [E.Var(b.clone(), requires_grad=True) for b in biases]
    tape = E.Tape()
    with E.recording(tape):
        if fused:
            assert ops.mlp_fusable(x, widths)
            out = ops.mlp(x, Ws, bs)
        else:
            out = x
            for W, b in zip(Ws, bs):
                out = ops.dense(out, W, b, "relu")
    out.requires_grad = True
    E.add_grad(out, gy)
    tape.backward()
    torch.cuda.synchronize()
    return out.data, x.grad, [W.grad for W in Ws], [b.grad for b in bs]


def test_mlp_random_against_float64_and_per_layer(cuda, gen):
    """845 -> (256, 128, 64) at B = 8192: forward output and the x, W, b gradients of ops.mlp and of the per-layer
    path, each within the split-bf16 bound of float64 (relu masks from float64; an element whose pre-activation is
    within the forward bound of 0 may take either side, and its full gradient is added to the bound)."""
    B, dims = 8192, [845, 256, 128, 64]
    x = torch.randn((B, 845), generator=gen, device=cuda)
    Ws = [torch.randn((dims[i], dims[i + 1]), generator=gen, device=cuda) * dims[i] ** -0.5 for i in range(3)]
    bs = [torch.randn((dims[i + 1],), generator=gen, device=cuda) * 0.1 for i in range(3)]
    gy = torch.randn((B, 64), generator=gen, device=cuda)

    def eps(k):
        return (k + 16) * U + 2.0 ** -15

    # float64 forward with an error chain
    h, habs, err, pres, errs, hs = x.double(), x.double().abs(), None, [], [], [x.double()]
    for i in range(3):
        W, b = Ws[i].double(), bs[i].double()
        pre = h @ W + b
        a = habs @ W.abs() + b.abs()
        e = eps(dims[i]) * a + (err @ W.abs() if err is not None else 0.0)
        pres.append(pre)
        errs.append(e)
        h, habs, err = torch.relu(pre), a, e
        hs.append(h)
    # float64 backward with an error chain; ambiguous masks add the full gradient to the bound
    g, gabs, gerr = gy.double(), gy.double().abs(), torch.zeros_like(gy, dtype=torch.float64)
    ref_dw, bnd_dw, ref_db, bnd_db = [None] * 3, [None] * 3, [None] * 3, [None] * 3
    for i in reversed(range(3)):
        mask = (pres[i] > 0).double()
        amb = (pres[i].abs() <= errs[i]).double()
        dz, dzabs, dzerr = g * mask, gabs * mask, gerr * mask + gabs * amb
        hin = hs[i]
        ref_dw[i] = hin.t() @ dz
        bnd_dw[i] = eps(B) * (hin.abs().t() @ dzabs) + hin.abs().t() @ dzerr + \
            (errs[i - 1].t() @ dzabs if i > 0 else 0.0)
        ref_db[i] = dz.sum(0)
        bnd_db[i] = (B + 16) * U * dzabs.sum(0) + dzerr.sum(0)
        W = Ws[i].double()
        g, gabs, gerr = dz @ W.t(), dzabs @ W.abs().t(), eps(dims[i + 1]) * (dzabs @ W.abs().t()) + dzerr @ W.abs().t()
    ref_dx, bnd_dx = g, gerr

    results = {f: _run_dnn(x, dims[1:], Ws, bs, gy, f) for f in (True, False)}
    for fused, (y, dx, dws, dbs) in results.items():
        tag = "fused" if fused else "per-layer"
        _within(y, hs[-1], errs[-1], tag + " forward")
        _within(dx, ref_dx, bnd_dx, tag + " dx")
        for i in range(3):
            _within(dws[i], ref_dw[i], bnd_dw[i], tag + " dW_%d" % i)
            _within(dbs[i], ref_db[i], bnd_db[i], tag + " db_%d" % i)


def _within(got, ref, bound, what):
    err = (got.double() - ref).abs()
    assert bool(torch.isfinite(got).all()), what
    ok = err <= bound + 1e-30
    assert bool(ok.all()), "%s: %d elements out of bound, worst %.3e" % (what, int((~ok).sum()),
                                                                        float((err - bound).max()))


# ---- selection in DNN.call ---------------------------------------------------------------------------------------
def _dnn_calls(monkeypatch, B=512, kdim=64, hidden=(256, 128, 64), training=False, **kw):
    L, K, ops, E = _mods()
    from deepctr_b200.layers.core import DNN
    calls = []
    real = ops.mlp
    monkeypatch.setattr(ops, "mlp", lambda *a: calls.append(1) or real(*a))
    layer = DNN(hidden, **kw)
    layer._maybe_build((None, kdim))
    x = E.Var(torch.randn((B, kdim), device="cuda"), requires_grad=True)
    out = layer.call(x, training=training)
    assert tuple(out.data.shape) == (B, hidden[-1])
    return len(calls)


def test_dnn_takes_fused_path(cuda, monkeypatch):
    assert _dnn_calls(monkeypatch) == 1
    assert _dnn_calls(monkeypatch, output_activation="relu", dropout_rate=0.5, training=False) == 1


@pytest.mark.parametrize("case", ["fp32", "bn", "dropout", "sigmoid", "width", "small_batch", "one_layer"])
def test_dnn_fallbacks(cuda, monkeypatch, case):
    L, K, ops, E = _mods()
    kw = {}
    if case == "fp32":
        ops.set_gemm_precision("fp32")
    try:
        if case == "bn":
            kw = dict(use_bn=True)
        elif case == "dropout":
            kw = dict(dropout_rate=0.5, training=True)
        elif case == "sigmoid":
            kw = dict(output_activation="sigmoid")
        elif case == "width":
            kw = dict(hidden=(256, 96, 64))
        elif case == "small_batch":
            kw = dict(B=127)
        elif case == "one_layer":
            kw = dict(hidden=(256,))
        assert _dnn_calls(monkeypatch, **kw) == 0
    finally:
        ops.set_gemm_precision("bf16x3")
