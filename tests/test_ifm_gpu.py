"""GPU: the field-weight kernels of IFM / DIFM, and the two builders.

* b2ctr_fm_weighted_fwd / _bwd, b2ctr_field_scale_fwd / _bwd and b2ctr_softmax_rows_fwd / _bwd against float64 over
  F = 1 / 2 / 26 / 64 and E = 1 / 4 / 5 / 32 / 64, with x and m windows of wider buffers, m with zeros and negative
  entries, dx written into a window of a wider buffer and added to a non-zero gradient (accumulate), and batches that
  are not a multiple of a CTA's samples;
* the C2 shape (B = 65536, F = 26, E = 32): x a window of the [B, 848] gather buffer;
* fm_weighted with m == 1 equals b2ctr_fm_fwd / _bwd bit for bit; the backwards are bit-identical from run to run;
* the IFM step runs fm_weighted and materialises no [B, F, E] product; a refine product consumed by Flatten -> Dense
  as well as FM is materialised and has the right gradients; the reference test's dnn_dropout=0.5 configurations
  train with a finite loss.
Model fixtures (with model_golden_checks): logits and one SGD step in both GEMM precisions; a graph-replayed IFM /
DIFM step equals an eager one.
"""
import numpy as np
import pytest
import torch

import b2_helpers as H
import model_golden_checks as C

pytestmark = pytest.mark.gpu

T = C.gpu_model_tests("ifm")
test_model_forward_matches_reference = T.forward
test_model_sgd_step_matches_reference_gradients = T.sgd_step
test_graph_replayed_step_equals_eager = C.graph_replay_test([
    pytest.param("IFM", dict(dnn_hidden_units=(32, 16)), id="ifm"),
    pytest.param("DIFM", dict(dnn_hidden_units=(32,), att_head_num=2), id="difm")])


def _operands(cuda, B, F, E, seed, ldx=None, x0=2):
    """x a [B, F*E] window at column x0 of a [B, ldx] buffer; m a [B, F] window at column 1 of a [B, F + 3] buffer,
    with zeros and negative entries."""
    rng = np.random.RandomState(seed)
    ldx = ldx or x0 + F * E + 7
    buf = torch.tensor(rng.normal(0, 0.5, size=(B, ldx)).astype(np.float32), device=cuda)
    mv = rng.normal(0, 1.0, size=(B, F + 3)).astype(np.float32)
    mv[rng.rand(B, F + 3) < 0.1] = 0.0
    mbuf = torch.tensor(mv, device=cuda)
    return rng, buf, buf[:, x0:x0 + F * E], ldx, mbuf[:, 1:1 + F]


def _fm64(x, m):
    y = x * m.unsqueeze(-1)
    return 0.5 * (y.sum(1) ** 2 - (y * y).sum(1)).sum(1)


def _check_fm(cuda, B, F, E, seed, ldx=None, x0=2, chunk=8192):
    from deepctr_b200 import kernels as K
    rng, buf, xw, ldx, m = _operands(cuda, B, F, E, seed, ldx, x0)
    out = K.fm_weighted_fwd(xw, ldx, m, F, E, B)
    g = torch.tensor(rng.normal(0, 1.0, size=B).astype(np.float32), device=cuda)
    # dx into a window of a wider buffer that already holds a gradient (accumulate); the rest must stay untouched
    dbuf = torch.tensor(rng.normal(0, 1.0, size=(B, F * E + 9)).astype(np.float32), device=cuda)
    d0 = dbuf.clone()
    dxw = dbuf[:, 4:4 + F * E]
    _, dm = K.fm_weighted_bwd(xw, ldx, m, F, E, g, B, dx=dxw, accumulate=True)
    assert torch.equal(dbuf[:, :4], d0[:, :4]) and torch.equal(dbuf[:, 4 + F * E:], d0[:, 4 + F * E:])
    for b0 in range(0, B, chunk):
        sl = slice(b0, min(B, b0 + chunk))
        x64 = xw[sl].double().reshape(-1, F, E).requires_grad_(True)
        m64 = m[sl].double().requires_grad_(True)
        ref = _fm64(x64, m64)
        (ref * g[sl].double()).sum().backward()
        with torch.no_grad():
            y = (x64 * m64.unsqueeze(-1)).abs()
            ga = g[sl].double().abs()
            sq = float((y * y).sum((1, 2)).max())
            fdx = float((ga[:, None, None] * m64.abs().unsqueeze(-1) * y.sum(1, keepdim=True)).max())
            fdm = float((ga[:, None] * (x64.abs() * y.sum(1, keepdim=True)).sum(2)).max())
        H.close(out[sl], ref.detach(), "fm_weighted out", 5e-5, floor=sq)
        H.close((dxw[sl] - d0[sl, 4:4 + F * E]).reshape(-1, F, E), x64.grad, "fm_weighted dx", 1e-4, floor=fdx)
        H.close(dm[sl], m64.grad, "fm_weighted dm", 1e-4, floor=fdm)
    return xw, ldx, m, g


def _check_scale(cuda, B, F, E, seed):
    from deepctr_b200 import kernels as K
    rng, buf, xw, ldx, m = _operands(cuda, B, F, E, seed)
    yb = torch.full((B, F * E + 6), 7.0, device=cuda)
    y = K.field_scale_fwd(xw, ldx, m, F, E, B, out=yb[:, 3:3 + F * E])
    assert bool((yb[:, :3] == 7.0).all()) and bool((yb[:, 3 + F * E:] == 7.0).all())
    x64, m64 = xw.double().reshape(B, F, E).requires_grad_(True), m.double().requires_grad_(True)
    ref = x64 * m64.unsqueeze(-1)
    H.close(y.reshape(B, F, E), ref.detach(), "field_scale y", 1e-7)
    gb = torch.tensor(rng.normal(0, 1.0, size=(B, F * E + 5)).astype(np.float32), device=cuda)
    g = gb[:, 5:]
    dbuf = torch.tensor(rng.normal(0, 1.0, size=(B, F * E + 2)).astype(np.float32), device=cuda)
    d0 = dbuf.clone()
    _, dm = K.field_scale_bwd(g, xw, ldx, m, F, E, B, dx=dbuf[:, 1:1 + F * E], accumulate=True)
    (ref * g.double().reshape(B, F, E)).sum().backward()
    H.close((dbuf[:, 1:1 + F * E] - d0[:, 1:1 + F * E]).reshape(B, F, E), x64.grad, "field_scale dx", 5e-5)
    assert torch.equal(dbuf[:, 0], d0[:, 0]) and torch.equal(dbuf[:, -1], d0[:, -1])
    H.close(dm, m64.grad, "field_scale dm", 1e-5)
    dx2, dm2 = K.field_scale_bwd(g, xw, ldx, m, F, E, B)
    H.close(dx2.reshape(B, F, E), x64.grad, "field_scale dx (overwrite)", 1e-7)
    _, dm3 = K.field_scale_bwd(g, xw, ldx, m, F, E, B, want_dx=False)
    assert torch.equal(dm2, dm) and torch.equal(dm3, dm)


FS = [1, 2, 26, 64]
ES = [1, 4, 5, 32, 64]


@pytest.mark.parametrize("E", ES)
@pytest.mark.parametrize("F", FS)
def test_fm_weighted_matches_float64(cuda, F, E):
    _check_fm(cuda, 1001 if F * E < 64 * 64 else 203, F, E, 11 * F + E)


@pytest.mark.parametrize("E", ES)
@pytest.mark.parametrize("F", FS)
def test_field_scale_matches_float64(cuda, F, E):
    _check_scale(cuda, 1001 if F * E < 64 * 64 else 203, F, E, 13 * F + E)


@pytest.mark.parametrize("scale", [1.0, 26.0])
@pytest.mark.parametrize("C", FS + [100])
def test_softmax_rows_matches_float64(cuda, C, scale):
    from deepctr_b200 import kernels as K
    B = 1001
    rng = np.random.RandomState(C)
    xb = torch.tensor(rng.normal(0, 3.0, size=(B, C + 5)).astype(np.float32), device=cuda)
    xb[:, 2] += 60.0            # large logits: the maximum is subtracted first
    x = xb[:, 2:2 + C]
    y = K.softmax_rows_fwd(x, scale)
    x64 = x.double().requires_grad_(True)
    ref = scale * torch.softmax(x64, dim=1)
    H.close(y, ref.detach(), "softmax y", 1e-6)
    gb = torch.tensor(rng.normal(0, 1.0, size=(B, C + 3)).astype(np.float32), device=cuda)
    g = gb[:, 3:]
    dx = K.softmax_rows_bwd(y, g, scale)
    (ref * g.double()).sum().backward()
    H.close(dx, x64.grad, "softmax dx", 1e-5, floor=float((ref.detach().abs() * g.double().abs()).max()))


def test_kernels_at_c2_shape(cuda):
    """B = 65536, F = 26, E = 32: x the embedding window of the [B, 848] gather buffer (832 embedding + 13 dense
    columns, padded to 848)."""
    _check_fm(cuda, 65536, 26, 32, 3, ldx=848, x0=0)


def test_unit_weights_give_fm_bit_for_bit(cuda):
    from deepctr_b200 import kernels as K
    for B, F, E in ((4099, 26, 32), (1001, 7, 5), (203, 64, 64), (513, 1, 1)):
        _, buf, xw, ldx, _ = _operands(cuda, B, F, E, F + E)
        ones = torch.ones((B, F), device=cuda)
        assert torch.equal(K.fm_weighted_fwd(xw, ldx, ones, F, E, B), K.fm_fwd(xw, F, E, ldx))
        g = torch.randn(B, device=cuda)
        dx, _ = K.fm_weighted_bwd(xw, ldx, ones, F, E, g, B)
        assert torch.equal(dx, K.fm_bwd(xw, F, E, g, dx=torch.empty((B, F * E), device=cuda), ldx=ldx))
        base = torch.randn((B, F * E), device=cuda)
        a, b = base.clone(), base.clone()
        K.fm_weighted_bwd(xw, ldx, ones, F, E, g, B, dx=a, accumulate=True)
        K.fm_bwd(xw, F, E, g, dx=b, accumulate=True, ldx=ldx)
        assert torch.equal(a, b)


def test_backwards_are_deterministic(cuda):
    from deepctr_b200 import kernels as K
    B, F, E = 4099, 26, 32
    xw, ldx, m, g = _check_fm(cuda, B, F, E, 5)
    dx, dm = K.fm_weighted_bwd(xw, ldx, m, F, E, g, B)
    for _ in range(2):
        dx2, dm2 = K.fm_weighted_bwd(xw, ldx, m, F, E, g, B)
        assert torch.equal(dx, dx2) and torch.equal(dm, dm2)
    y = K.softmax_rows_fwd(m, 26.0)
    gy = torch.randn_like(y)
    assert torch.equal(K.softmax_rows_bwd(y, gy, 26.0), K.softmax_rows_bwd(y, gy, 26.0))


def test_ifm_step_runs_fm_weighted_and_writes_no_refined_block(cuda, monkeypatch):
    """The refined FM input m ⊙ x reaches FM as its factors: the step launches fm_weighted forward and backward, and
    the only materialised field scale is the dim-1 one of the linear lookups."""
    from deepctr_b200 import kernels as K
    calls = []
    for name in ("fm_weighted_fwd", "fm_weighted_bwd", "field_scale_fwd", "fm_fwd"):
        real = getattr(K, name)

        def spy(*a, _real=real, _name=name, **kw):
            calls.append((_name, a[4] if _name == "field_scale_fwd" else None))
            return _real(*a, **kw)
        monkeypatch.setattr(K, name, spy)
    H.train("IFM", "off", dict(dnn_hidden_units=(16,)), steps=2)
    names = [c[0] for c in calls]
    assert names.count("fm_weighted_fwd") == 2 and names.count("fm_weighted_bwd") == 2, names
    assert "fm_fwd" not in names
    assert [d for n, d in calls if n == "field_scale_fwd"] == [1, 1]


def test_refine_product_feeding_other_layers_is_materialised(cuda):
    """A refine Lambda consumed by Flatten -> Dense and by FM: the Dense reads the materialised product, FM its
    factors; the loss and every gradient of one SGD step match a torch restatement."""
    from deepctr_b200 import engine as E, ops
    from deepctr_b200.engine import Dense, Flatten, Lambda, SGD
    from deepctr_b200.feature_column import build_input_features, input_from_feature_columns
    from deepctr_b200.layers.core import PredictionLayer
    from deepctr_b200.layers.interaction import FM
    from deepctr_b200.layers.utils import add_func, concat_func
    from oracle import ops as O
    rng = np.random.RandomState(9)
    cols, x, y = H.criteo_like(rng, 256, n_sparse=10)
    cols = cols[:10]
    E.clear_session()
    features = build_input_features(cols)
    embs, _ = input_from_feature_columns(features, cols, 0, 1024)
    fm_in = concat_func(embs, axis=1)
    m = Dense(10, use_bias=False)(Flatten()(fm_in))
    refined = Lambda(lambda v: ops.scale_fields(v[0], v[1]))([fm_in, m])
    logit = add_func([Dense(1, use_bias=False)(Flatten()(refined)), FM()(refined)])
    model = E.Model(list(features.values()), PredictionLayer("binary")(logit))
    w0 = {w.name: torch.tensor(w.value(), requires_grad=True) for w in model.weights}
    lr = 0.5
    model.compile(SGD(lr), "binary_crossentropy", embedding_update="dense")
    loss = model.train_on_batch({k: v for k, v in x.items() if k in features}, y)
    # torch restatement
    xe = torch.stack([w0["sparse_emb_C%d/embeddings" % i][torch.as_tensor(x["C%d" % i].astype(np.int64))]
                      for i in range(10)], dim=1)
    dense_names = sorted(k for k in w0 if k.startswith("dense"))
    mw = xe.flatten(1) @ w0[dense_names[0]]
    r = xe * mw.unsqueeze(-1)
    lg = r.flatten(1) @ w0[dense_names[1]] + O.fm(r)
    bias = [v for k, v in w0.items() if k.endswith("/global_bias")]
    pred = O.prediction(lg, bias[0] if bias else None, "binary")
    ref_loss = O.binary_crossentropy(y, pred)
    ref_loss.backward()
    want_loss = float(ref_loss.detach())
    assert abs(loss - want_loss) <= 1e-4 * max(1.0, abs(want_loss)), (loss, want_loss)
    for w in model.weights:
        want = w0[w.name].grad.numpy()
        got = (w0[w.name].detach().numpy() - w.value()) / lr
        np.testing.assert_allclose(got, want, rtol=2e-3, atol=3e-4 * float(np.abs(want).max()) + 2e-6, err_msg=w.name)


def test_reference_test_configurations_train_with_dropout(cuda):
    """The reference's tests/models/IFM_test.py / DIFM_test.py configurations: dnn_hidden_units (4,) and (4, 4),
    dnn_dropout=0.5; a few steps of training give finite losses."""
    from deepctr_b200 import engine as E, models as M
    from deepctr_b200.engine import SGD
    for builder in ("IFM", "DIFM"):
        for hidden in ((4,), (4, 4)):
            cols, x, y = H.criteo_like(np.random.RandomState(6), 512, n_sparse=10)
            E.clear_session()
            model = getattr(M, builder)(cols, cols, dnn_hidden_units=hidden, dnn_dropout=0.5, l2_reg_linear=0,
                                        l2_reg_embedding=0)
            model.compile(SGD(0.05), "binary_crossentropy", embedding_update="sparse")
            losses = [model.train_on_batch(x, y) for _ in range(3)]
            assert np.isfinite(losses).all(), (builder, hidden, losses)
