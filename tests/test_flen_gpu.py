"""GPU: FLEN's field-wise bi-interaction kernels and the FLEN builder.

* b2ctr_field_wise_bi_fwd / _bwd against float64 over 2 to 8 groups, group sizes 1 to 5, E = 1, 3, 4, 5, 16 and
  32, interleaved and contiguous members, windows that are or are not 16-byte aligned, dx written or added, and
  use_bias both ways; at the C2 bench shape (B = 65536, 26 fields, E = 32, dx added into a [B, 848] buffer);
* the backward is bit-identical from run to run; shapes outside the limits raise ValueError naming them;
* a planned FLEN forward is one field_wise_bi_fwd launch, a training step one field_wise_bi_bwd, and with contiguous
  groups the forward copies none of the group inputs;
* the reference's examples/run_flen.py flow on its own Avazu sample, against the CPU oracle trained with the same
  Keras semantics.
Fixtures (with model_golden_checks): the FieldWiseBiInteraction layer fixtures and the model fixtures' logits and
one SGD step in both GEMM precisions.
"""
import os

import numpy as np
import pytest
import torch

import b2_helpers as H
import model_golden_checks as C
import flen_family  # noqa: F401  (registers the "flen" fixture families)
import flen_oracle as FO
from oracle import ops as O

pytestmark = pytest.mark.gpu
DATA = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "avazu_sample.txt")

T = C.gpu_model_tests("flen")
test_model_forward_matches_reference = T.forward
test_model_sgd_step_matches_reference_gradients = T.sgd_step
test_layer_fixture = C.gpu_layer_test("flen")


def _case(cuda, sizes, E, B, interleave=True, offset=0, use_bias=True, accumulate=False, extra=3, seed=0):
    """Fields of ``sizes`` groups laid out in a [B, ld] buffer (group of field f = its position among the groups'
    members, interleaved or contiguous) from column ``offset``; runs the forward and the backward and returns
    (h, dh, weight gradients, dx buffer before, dx buffer after, float64 reference values)."""
    from deepctr_b200 import kernels as K
    g = torch.Generator(device=cuda).manual_seed(seed)
    G = len(sizes)
    order = [k for k in range(G) for _ in range(sizes[k])]
    if interleave:
        order = [k for r in range(max(sizes)) for k in range(G) if r < sizes[k]]
    F = len(order)
    ld = offset + F * E + extra
    x = torch.randn((B, ld), generator=g, device=cuda) * 0.5
    cols = [offset + f * E for f in range(F)]
    P = G * (G - 1) // 2
    kmf = torch.randn((P, 1), generator=g, device=cuda) * 0.5 + 1.0
    kfm = torch.randn((G, 1), generator=g, device=cuda) * 0.2 + 0.5
    bmf = torch.randn((E,), generator=g, device=cuda) if use_bias else None
    bfm = torch.randn((E,), generator=g, device=cuda) if use_bias else None
    out = torch.full((B, E + 2), 7.0, device=cuda)
    K.field_wise_bi_fwd(x, cols, order, G, E, B, kmf, kfm, bmf, bfm, out, outcol=1)
    dh = torch.randn((B, E), generator=g, device=cuda)
    dbuf = torch.randn((B, ld), generator=g, device=cuda) if accumulate else torch.full((B, ld), 3.0, device=cuda)
    before = dbuf.clone()
    dws = K.field_wise_bi_bwd(x, cols, order, G, E, B, kmf, kfm, bmf, bfm, dh, dx=dbuf, dx_accumulate=accumulate,
                              want_dkernel=(True, True), want_dbias=(use_bias, use_bias))
    # float64 reference
    xd = x.double().requires_grad_(True)
    groups = [torch.stack([xd[:, c:c + E] for c, k in zip(cols, order) if k == grp], dim=1) for grp in range(G)]
    w64 = [v.double().requires_grad_(True) if v is not None else None for v in (kmf, kfm, bmf, bfm)]
    want = FO.field_wise_bi(groups, *w64)
    (want * dh.double()).sum().backward()
    # the size of the terms each weight gradient sums: sum_{b,e} |dh| * max_g (S_g^2 + Q_g).  A one-member group
    # has S^2 - Q = 0 exactly, which fp32 reaches only to rounding of these terms.
    with torch.no_grad():
        sq = torch.stack([g.sum(1) ** 2 + (g * g).sum(1) for g in groups], 1).amax(1)
        mag = float((dh.double().abs() * sq).sum())
    return out, dws, before, dbuf, want.detach(), xd.grad, w64, cols, mag


def _check(cuda, sizes, E, B=300, **kw):
    out, dws, before, dbuf, want, gx, w64, cols, mag = _case(cuda, sizes, E, B, **kw)
    scale = float(want.abs().max())
    torch.testing.assert_close(out[:, 1:1 + E].double(), want, rtol=1e-5, atol=1e-5 * scale)
    assert torch.all(out[:, 0] == 7.0) and torch.all(out[:, E + 1] == 7.0)
    expect = before.double().clone()
    fieldcols = torch.zeros(before.shape[1], dtype=torch.bool, device=cuda)
    for c in cols:
        fieldcols[c:c + E] = True
    if kw.get("accumulate"):
        expect[:, fieldcols] += gx[:, fieldcols]
    else:
        expect[:, fieldcols] = gx[:, fieldcols]
    gscale = float(gx.abs().max())
    torch.testing.assert_close(dbuf.double(), expect, rtol=1e-5, atol=1e-5 * gscale)
    assert torch.equal(dbuf[:, ~fieldcols], before[:, ~fieldcols])
    for got, w in zip(dws, w64):
        if w is None:
            assert got is None
            continue
        torch.testing.assert_close(got.double().reshape(w.shape), w.grad, rtol=1e-4,
                                   atol=1e-5 * float(w.grad.abs().max()) + 1e-6 * mag)


@pytest.mark.parametrize("sizes", [(1, 1), (2, 3), (1, 4, 2), (3, 3, 3), (5, 1), (1, 2, 1, 3, 1, 1, 2, 1),
                                   (2,) * 8])
@pytest.mark.parametrize("E", [1, 3, 4, 16])
def test_kernels_match_float64(cuda, sizes, E):
    _check(cuda, sizes, E)


@pytest.mark.parametrize("E,offset,interleave,use_bias,accumulate", [
    (4, 0, True, True, True), (4, 1, True, False, True), (5, 0, False, True, False), (16, 2, False, False, True),
    (32, 0, True, True, False), (32, 3, True, True, True), (1, 0, True, False, True)])
def test_layouts_bias_and_accumulation_match_float64(cuda, E, offset, interleave, use_bias, accumulate):
    _check(cuda, (3, 2, 4), E, B=517, offset=offset, interleave=interleave, use_bias=use_bias,
           accumulate=accumulate)


def test_c2_bench_shape(cuda):
    """26 fields in groups i % 3, E = 32, B = 65536, dx added into the gather-buffer-shaped [B, 848] buffer."""
    _check(cuda, (9, 9, 8), 32, B=65536, extra=848 - 26 * 32, accumulate=True)


def test_backward_is_deterministic(cuda):
    from deepctr_b200 import kernels as K
    B, E, G = 200000, 16, 3
    g = torch.Generator(device=cuda).manual_seed(5)
    x = torch.randn((B, 21 * E), generator=g, device=cuda)
    cols, order = [f * E for f in range(21)], [f % G for f in range(21)]
    kmf, kfm = torch.ones((3, 1), device=cuda), torch.full((3, 1), 0.5, device=cuda)
    bmf = bfm = torch.zeros((E,), device=cuda)
    dh = torch.randn((B, E), generator=g, device=cuda)
    runs = []
    for _ in range(2):
        dx = torch.zeros_like(x)
        dws = K.field_wise_bi_bwd(x, cols, order, G, E, B, kmf, kfm, bmf, bfm, dh, dx=dx, dx_accumulate=True,
                                  want_dkernel=(True, True), want_dbias=(True, True))
        runs.append([dx] + list(dws))
    for a, b in zip(*runs):
        assert torch.equal(a, b)


@pytest.mark.parametrize("shapes,limit", [([(1, 4)] * 9, "FWBI_MAX_GROUPS"),
                                          ([(200, 4), (57, 4)], "FWBI_MAX_FIELDS"),
                                          ([(1, 257), (1, 257)], "FWBI_MAX_DIM")])
def test_shapes_outside_the_limits_raise(cuda, shapes, limit):
    from deepctr_b200 import engine as E, ops
    xs = [E.Var(torch.zeros((4,) + s, device=cuda)) for s in shapes]
    w = torch.ones((len(shapes) * (len(shapes) - 1) // 2, 1), device=cuda)
    with pytest.raises(ValueError, match=limit):
        ops.field_wise_bi([[v] for v in xs], E.Var(w), E.Var(torch.ones((len(shapes), 1), device=cuda)))


def _flen_model(groups, n=512, V=40, E=8, **kw):
    from deepctr_b200 import engine as E_, models as M
    from deepctr_b200.feature_column import SparseFeat
    rng = np.random.RandomState(3)
    cols = [SparseFeat("C%d" % i, V, E, group_name=gname) for i, gname in enumerate(groups)]
    x = {"C%d" % i: rng.randint(0, V, size=n).astype(np.int32) for i in range(len(groups))}
    y = (rng.rand(n) < 0.3).astype(np.float32)
    E_.clear_session()
    return M.FLEN(cols, cols, l2_reg_embedding=0, l2_reg_linear=0, dnn_hidden_units=(16,), **kw), x, y


def _launches(model, x, y):
    from deepctr_b200 import kernels as K
    from deepctr_b200.engine import SGD
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
    return fwd, step


@pytest.mark.parametrize("groups", [[str(i % 3) for i in range(9)], [str(i // 3) for i in range(9)]],
                         ids=["interleaved", "contiguous"])
def test_one_launch_forward_and_backward(cuda, groups):
    model, x, y = _flen_model(groups)
    fwd, step = _launches(model, x, y)
    assert fwd.get("field_wise_bi_fwd") == 1 and "field_wise_bi_bwd" not in fwd, fwd
    assert step.get("field_wise_bi_fwd") == 1 and step.get("field_wise_bi_bwd") == 1, step
    if groups[1] == "0":
        # contiguous groups: the only copies are concat([h, DNN output]) before the last Dense
        assert fwd.get("copy2d", 0) <= 2, fwd


def _avazu():
    import pandas as pd
    from sklearn.model_selection import train_test_split
    from sklearn.preprocessing import LabelEncoder
    from deepctr_b200.feature_column import SparseFeat, get_feature_names
    data = pd.read_csv(DATA)
    data['day'] = data['hour'].apply(lambda v: str(v)[4:6])
    data['hour'] = data['hour'].apply(lambda v: str(v)[6:])
    sparse = ['hour', 'C1', 'banner_pos', 'site_id', 'site_domain', 'site_category', 'app_id', 'app_domain',
              'app_category', 'device_id', 'device_model', 'device_type', 'device_conn_type', 'C14', 'C15', 'C16',
              'C17', 'C18', 'C19', 'C20', 'C21']
    data[sparse] = data[sparse].fillna('-1', )
    for feat in sparse:
        data[feat] = LabelEncoder().fit_transform(data[feat])
    info = dict(C14='user', C15='user', C16='user', C17='user', C18='user', C19='user', C20='user', C21='user',
                C1='user', banner_pos='context', site_id='context', site_domain='context', site_category='context',
                app_id='item', app_domain='item', app_category='item', device_model='user', device_type='user',
                device_conn_type='context', hour='context', device_id='user')
    cols = [SparseFeat(f, vocabulary_size=int(data[f].max()) + 1, embedding_dim=16, use_hash=False, dtype='int32',
                       group_name=info[f]) for f in sparse]
    names = get_feature_names(cols + cols)
    train, test = train_test_split(data, test_size=0.2, random_state=2020)
    return cols, names, train, test


def _oracle_w(model, requires_grad):
    from deepctr_b200.layers import FieldWiseBiInteraction
    W = H.oracle_weights(model, requires_grad=requires_grad)
    (layer,) = [l for l in model.layers if isinstance(l, FieldWiseBiInteraction)]
    W["fwbi"] = [torch.tensor(w.value(), requires_grad=requires_grad)
                 for w in (layer.kernel_mf, layer.kernel_fm, layer.bias_mf, layer.bias_fm)]
    W["dnn_bn"] = None
    return W


@pytest.mark.usefixtures("gemm_precision")
def test_run_flen_avazu_sample_training_matches_oracle(cuda):
    from deepctr_b200.models import FLEN
    cols, names, train, test = _avazu()
    assert len(cols) == 21 and len(train) == 80 and len(test) == 20
    x_tr = {n: train[n] for n in names}
    y_tr = train[['click']].values
    x_te = {n: test[n] for n in names}
    model = FLEN(cols, cols, task='binary')               # reference defaults: l2 1e-5, dnn (256, 128, 64)
    H.randomize_weights(model, np.random.RandomState(0), 0.05)
    model.compile("adam", "binary_crossentropy", metrics=['binary_crossentropy'], embedding_update="dense")
    W = _oracle_w(model, True)
    leaves = H.flat_params(W)
    l2 = {n: (1e-5 if (n.startswith("tables/") or n == "linear_kernel") else 0.0) for n in leaves}
    m = {n: torch.zeros_like(t) for n, t in leaves.items()}
    v = {n: torch.zeros_like(t) for n, t in leaves.items()}
    x_te_np = {n: np.asarray(x_te[n]) for n in names}
    with torch.no_grad():
        _, want0 = FO.flen(x_te_np, cols, cols, W)
    assert H.rel_err(model.predict(x_te, batch_size=256), want0.numpy()) < 1e-4
    split = int(len(y_tr) * 0.8)                          # validation_split=0.2 takes the LAST 20 %
    xo = {n: np.asarray(x_tr[n])[:split] for n in names}
    yo = y_tr[:split].reshape(-1)
    epochs, want_losses = 10, []
    for step in range(1, epochs + 1):
        _, pred = FO.flen(xo, cols, cols, W)
        data_loss = O.binary_crossentropy(yo, pred)
        data_loss.backward()
        reg = sum(l2[n] * float((t.detach().double() ** 2).sum()) for n, t in leaves.items())
        want_losses.append(float(data_loss) + reg)
        with torch.no_grad():
            lr_t = 1e-3 * np.sqrt(1 - 0.999 ** step) / (1 - 0.9 ** step)
            for n, t in leaves.items():
                if t.grad is None:
                    continue
                g = t.grad + 2 * l2[n] * t
                m[n] = 0.9 * m[n] + 0.1 * g
                v[n] = 0.999 * v[n] + 0.001 * g * g
                t -= lr_t * m[n] / (v[n].sqrt() + 1e-7)
                t.grad = None
    hist = model.fit(x_tr, y_tr, batch_size=256, epochs=epochs, verbose=0, validation_split=0.2, shuffle=False)
    got = hist.history["loss"]
    assert len(got) == epochs and len(hist.history["val_loss"]) == epochs
    for a, b in zip(got, want_losses):
        assert abs(a - b) < 2e-3 * max(1.0, abs(b)), (got, want_losses)
    pred = model.predict(x_te, batch_size=256)
    _, want = FO.flen(x_te_np, cols, cols, W)
    assert pred.shape == (20, 1)
    assert H.rel_err(pred, want.detach().numpy()) < 2e-3
    from sklearn.metrics import log_loss
    assert np.isfinite(log_loss(test[['click']].values, pred.astype(np.float64), labels=[0, 1]))
