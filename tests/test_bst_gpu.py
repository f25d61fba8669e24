"""GPU: the fused attention and LayerNormalization kernels, the Transformer layer and the BST builder.

* b2ctr_mha_fwd / _bwd against a float64 restatement of deepctr/layers/sequence.py:544-617 over T = 1 / 7 / 50 / 128
  and (E, heads) = (8, 8) / (12, 4) / (64, 8) / (128, 2), lengths 0, 1 and T, separate query and key lengths or
  masks, blinding on and off, Q / K / V / residual read as windows of wider buffers, and a batch that is not a
  multiple of anything; the backward is bit-identical from run to run, and with dropout the output equals the
  restatement with the mask rebuilt from b2ctr_dropout;
* b2ctr_layernorm_fwd / _bwd against float64 with one and two summands, with and without gamma / beta;
* the Transformer layer (PositionEncoding, Q / K / V, attention, the shared LayerNormalization and the
  feed-forward) against a float64 restatement, in both GEMM precisions, for BST's, the reference test's and the
  default settings and for supports_masking=True: output, input gradients and every weight gradient;
* BST: a graph-replayed training step equals an eager one, 'sparse' and 'dense' embedding updates agree, and a
  C4-shaped step (B = 8192, T = 50, E = 64, 8 heads) trains.
"""
import numpy as np
import pytest
import torch

import b2_helpers as H

pytestmark = pytest.mark.gpu
PAD = -2.0 ** 32 + 1


def _close(got, want, what, tol=2e-5):
    want = want.detach().double() if isinstance(want, torch.Tensor) else torch.as_tensor(want, dtype=torch.float64)
    got = got.detach().double().cpu() if isinstance(got, torch.Tensor) else torch.as_tensor(got, dtype=torch.float64)
    want = want.cpu().reshape(got.shape)
    scale = max(float(want.abs().max()), 1e-30)
    err = float((got - want).abs().max()) / scale
    assert err < tol, "%s: max error %.3e relative to max |value|" % (what, err)


def ref_mha(q, k, v, heads, qvalid, kvalid, blinding, res=None, drop=None):
    """float64 restatement of sequence.py:544-617 on [B, T, W] projections; qvalid / kvalid bool [B, T]."""
    B, T, W = q.shape
    d = W // heads
    Q_, K_, V_ = (torch.cat(torch.split(t, d, dim=2), 0) for t in (q, k, v))          # [h*B, T, d]
    s = Q_ @ K_.transpose(1, 2) / d ** 0.5
    keep = kvalid.repeat(heads, 1)[:, None, :].expand(-1, T, -1)
    if blinding:
        keep = keep & ~torch.eye(T, dtype=torch.bool, device=q.device)[None]
    s = torch.where(keep, s, torch.full_like(s, PAD))
    s = s - s.max(-1, keepdim=True).values
    p = torch.softmax(s, -1) * qvalid.repeat(heads, 1)[:, :, None].double()
    if drop is not None:
        p = p * drop
    r = torch.cat(torch.split(p @ V_, B, 0), 2)
    return r + res if res is not None else r


def _valid(kind, B, T, rng, device):
    """int32 lengths [B] cycling through 0, 1, T and random values, or uint8 masks with an all-zero row."""
    if kind == "len":
        ln = np.array([[0, 1, T][i % 3] if i < 6 else rng.randint(0, T + 1) for i in range(B)], np.int32)
        t = torch.tensor(ln, device=device)
        return t, torch.arange(T, device=device)[None, :] < t[:, None]
    m = (rng.rand(B, T) < 0.6).astype(np.uint8)
    m[0] = 0
    m[1] = 1
    t = torch.tensor(m, device=device)
    return t, t.bool()


def _mha_case(cuda, B, T, E, heads, blinding, kind, rate=0.0, seed=0, seed_np=0):
    from deepctr_b200 import kernels as K
    rng = np.random.RandomState(seed_np)
    d = E // heads
    # q / k / v / residual are windows of one [B*T, 4E + 7] buffer
    ld = 4 * E + 7
    buf = torch.tensor(rng.normal(0, 1.0, size=(B * T, ld)).astype(np.float32), device=cuda)
    q, k, v, res = buf[:, 1:1 + E], buf[:, E + 2:2 * E + 2], buf[:, 2 * E + 4:3 * E + 4], buf[:, 3 * E + 6:4 * E + 6]
    qv, qvalid = _valid(kind, B, T, rng, cuda)
    kv, kvalid = _valid(kind, B, T, np.random.RandomState(seed_np + 1), cuda)
    kw = dict(qlen=qv, klen=kv) if kind == "len" else dict(qmask=qv, kmask=kv)
    scale = float(np.float32(1.0) / np.sqrt(np.float32(d)))
    out, stats = K.mha_fwd(q, ld, k, ld, v, ld, B, T, heads, d, scale, blinding=blinding, rate=rate, seed=seed,
                           res=res, ldr=ld, **kw)
    g = torch.tensor(rng.normal(0, 1.0, size=(B * T, E)).astype(np.float32), device=cuda)
    grads = K.mha_bwd(g, E, q, ld, k, ld, v, ld, stats, B, T, heads, d, scale, blinding=blinding, rate=rate,
                      seed=seed, **kw)
    drop = None
    if rate:
        ones = torch.ones((heads * B, T, T), dtype=torch.float32, device=cuda)
        drop = K.dropout(ones, rate, seed).double()
    ts = [t.double().reshape(B, T, E).requires_grad_(True) for t in (q, k, v, res)]
    ref = ref_mha(ts[0], ts[1], ts[2], heads, qvalid, kvalid, blinding, res=ts[3], drop=drop)
    (ref * g.double().reshape(B, T, E)).sum().backward()
    return out, grads, ref, ts, (q, k, v, g, stats, kw, scale, ld)


@pytest.mark.parametrize("kind", ["len", "mask"])
@pytest.mark.parametrize("blinding", [False, True])
@pytest.mark.parametrize("E,heads", [(8, 8), (12, 4), (64, 8), (128, 2)])
@pytest.mark.parametrize("T", [1, 7, 50, 128])
def test_mha_matches_float64(cuda, T, E, heads, blinding, kind):
    out, (dq, dk, dv), ref, ts, _ = _mha_case(cuda, 37, T, E, heads, blinding, kind)
    _close(out, ref, "out")
    _close(dq, ts[0].grad, "dq")
    _close(dk, ts[1].grad, "dk")
    _close(dv, ts[2].grad, "dv")


@pytest.mark.parametrize("T,E,heads", [(7, 12, 4), (50, 64, 8)])
def test_mha_dropout_uses_the_dropout_kernels_mask(cuda, T, E, heads):
    out, (dq, dk, dv), ref, ts, _ = _mha_case(cuda, 21, T, E, heads, False, "len", rate=0.3, seed=12345)
    _close(out, ref, "out")
    _close(dq, ts[0].grad, "dq")
    _close(dk, ts[1].grad, "dk")
    _close(dv, ts[2].grad, "dv")


def test_mha_backward_is_deterministic(cuda):
    from deepctr_b200 import kernels as K
    B, T, E, heads = 300, 50, 64, 8
    _, first, _, _, (q, k, v, g, stats, kw, scale, ld) = _mha_case(cuda, B, T, E, heads, False, "len")
    again = K.mha_bwd(g, E, q, ld, k, ld, v, ld, stats, B, T, heads, E // heads, scale, **kw)
    for a, b in zip(first, again):
        assert torch.equal(a, b)


def test_mha_rejects_unsupported_shapes(cuda):
    from deepctr_b200 import kernels as K
    x = torch.zeros((4 * 129, 8), device=cuda)
    with pytest.raises(ValueError):
        K.mha_fwd(x, 8, x, 8, x, 8, 4, 129, 1, 8, 1.0)
    y = torch.zeros((4 * 3, 65), device=cuda)
    with pytest.raises(ValueError):
        K.mha_fwd(y, 65, y, 65, y, 65, 4, 3, 1, 65, 1.0)


def _ln_case(cuda, rows, n, two, affine, seed=0):
    from deepctr_b200 import kernels as K
    rng = np.random.RandomState(seed)
    ld = n + 3
    buf = torch.tensor(rng.normal(0.5, 2.0, size=(rows, 2 * ld)).astype(np.float32), device=cuda)
    a, b = buf[:, :n], (buf[:, ld:ld + n] if two else None)
    gamma = torch.tensor(rng.normal(1, 0.3, size=n).astype(np.float32), device=cuda) if affine else None
    beta = torch.tensor(rng.normal(0, 0.3, size=n).astype(np.float32), device=cuda) if affine else None
    y, stats = K.layernorm_fwd(a, 2 * ld, b, 2 * ld, gamma, beta, rows, n, 1e-9)
    g = torch.tensor(rng.normal(size=(rows, n)).astype(np.float32), device=cuda)
    dx, dg, db = K.layernorm_bwd(a, 2 * ld, b, 2 * ld, gamma, stats, g, rows, n, want_dgamma=affine,
                                 want_dbeta=affine)
    x = (a.double() + (b.double() if two else 0)).requires_grad_(True)
    g64 = gamma.double().requires_grad_(True) if affine else None
    b64 = beta.double().requires_grad_(True) if affine else None
    mean = x.mean(-1, keepdim=True)
    ref = (x - mean) / torch.sqrt(((x - mean) ** 2).mean(-1, keepdim=True) + 1e-9)
    if affine:
        ref = ref * g64 + b64
    (ref * g.double()).sum().backward()
    return (y, dx, dg, db), (ref, x.grad, g64.grad if affine else None, b64.grad if affine else None), \
        (a, b, gamma, stats, g, ld)


@pytest.mark.parametrize("affine", [True, False])
@pytest.mark.parametrize("two", [False, True])
@pytest.mark.parametrize("n", [1, 8, 64, 100, 1024])
def test_layernorm_matches_float64(cuda, n, two, affine):
    got, want, _ = _ln_case(cuda, 37 * 7, n, two, affine)
    _close(got[0], want[0], "y", tol=1e-5)
    if n > 1:                      # n == 1: the normalised value is 0 and dx is rounding noise around 0
        _close(got[1], want[1], "dx", tol=1e-4)
    if affine:
        _close(got[2], want[2], "dgamma", tol=1e-5)
        _close(got[3], want[3], "dbeta", tol=1e-5)


def test_layernorm_backward_is_deterministic(cuda):
    from deepctr_b200 import kernels as K
    rows, n = 8192 * 50, 64
    got, _, (a, b, gamma, stats, g, ld) = _ln_case(cuda, rows, n, True, True)
    again = K.layernorm_bwd(a, 2 * ld, b, 2 * ld, gamma, stats, g, rows, n)
    for x, y in zip(got[1:], again):
        assert torch.equal(x, y)


# ---- the Transformer layer against a float64 restatement ------------------------------------------------------
def ref_transformer(X_q, X_k, W, cfg, qvalid, kvalid):
    """float64 restatement of Transformer.call (sequence.py:523-635) with dropout 0."""
    E = X_q.shape[-1]
    ln = lambda x: ((x - x.mean(-1, keepdim=True)) /
                    torch.sqrt(((x - x.mean(-1, keepdim=True)) ** 2).mean(-1, keepdim=True) + 1e-9)
                    * W["ln/gamma"] + W["ln/beta"])
    if cfg.get("use_positional_encoding", True):
        X_q = X_q + W["query_pe/lookup_table"] * E ** 0.5
        X_k = X_k + W["key_pe/lookup_table"] * E ** 0.5
    q, k, v = X_q @ W["query"], X_k @ W["key"], X_k @ W["value"]
    r = ref_mha(q, k, v, cfg["head_num"], qvalid, kvalid, cfg.get("blinding", True),
                res=X_q if cfg.get("use_res", True) else None)
    if cfg.get("use_layer_norm", False):
        r = ln(r)
    if cfg.get("use_feed_forward", True):
        fw2 = torch.relu(r @ W["fw1"]) @ W["fw2"]
        if cfg.get("use_res", True):
            r = r + fw2
        if cfg.get("use_layer_norm", False):
            r = ln(r)
    ot = cfg.get("output_type", "mean")
    if ot == "mean":
        return r.mean(1, keepdim=True)
    if ot == "sum":
        return r.sum(1, keepdim=True)
    return r


LAYER_CASES = {
    "bst": dict(att_embedding_size=4, head_num=2, use_layer_norm=True, blinding=False, output_type=None),
    "reference_test": dict(att_embedding_size=1, head_num=8, use_layer_norm=True, output_type="sum"),
    "defaults": dict(att_embedding_size=2, head_num=4),
    "masking": dict(att_embedding_size=4, head_num=2, use_layer_norm=True, supports_masking=True, output_type=None),
}


@pytest.mark.usefixtures("gemm_precision")
@pytest.mark.parametrize("name", sorted(LAYER_CASES))
def test_transformer_layer_matches_float64(cuda, name):
    from deepctr_b200 import engine as E
    from deepctr_b200.layers import Transformer
    cfg = LAYER_CASES[name]
    B, T = 37, 7
    Ed = cfg["att_embedding_size"] * cfg["head_num"]
    rng = np.random.RandomState(3)
    E.clear_session()
    layer = Transformer(seed=5, **cfg)
    Xq = torch.tensor(rng.normal(size=(B, T, Ed)).astype(np.float32), device=cuda)
    Xk = torch.tensor(rng.normal(size=(B, T, Ed)).astype(np.float32), device=cuda)
    ql = torch.tensor([[0, 1, T][i % 3] if i < 6 else rng.randint(0, T + 1) for i in range(B)], dtype=torch.int32,
                      device=cuda).reshape(B, 1)
    kl = torch.tensor(rng.randint(0, T + 1, size=(B, 1)).astype(np.int32), device=cuda)
    vq, vk = E.Var(Xq, requires_grad=True), E.Var(Xk, requires_grad=True)
    if cfg.get("supports_masking"):
        vq.mask = E.KMask(lengths=ql.reshape(-1), maxlen=T)
        vk.mask = E.KMask(lengths=kl.reshape(-1), maxlen=T)
        ins = [vq, vk]
    else:
        ins = [vq, vk, E.Var(ql), E.Var(kl)]
    layer._maybe_build(E._shape_of(ins))
    for w in layer.weights:          # O(1) weights so that every term matters
        if not w.name.endswith("lookup_table"):
            w.set_value(rng.normal(0, 0.5, size=w.shape).astype(np.float32))
        w.materialize()
    tape = E.Tape()
    with E.recording(tape):
        y = layer._invoke(ins, False)
    out = E.contiguous(y)
    gy = torch.tensor(rng.normal(size=tuple(out.shape)).astype(np.float32), device=cuda)
    y.requires_grad = True
    E.add_grad(y, gy)
    tape.backward()

    W = {w.name.split("/", 1)[1]: torch.tensor(w.value(), dtype=torch.float64, device=cuda, requires_grad=True)
         for w in layer.weights}
    x64 = [t.double().requires_grad_(True) for t in (Xq, Xk)]
    ar = torch.arange(T, device=cuda)[None, :]
    ref = ref_transformer(x64[0], x64[1], W, cfg, ar < ql, ar < kl)
    (ref * gy.double().reshape(ref.shape)).sum().backward()
    tol = 2e-4
    _close(out, ref, "out", tol)
    _close(vq.grad, x64[0].grad, "d queries", tol)
    _close(vk.grad, x64[1].grad, "d keys", tol)
    for w in layer.weights:
        key = w.name.split("/", 1)[1]
        if W[key].grad is None or not w.trainable:
            continue
        assert w.grad is not None, key
        _close(w.grad, W[key].grad, key, tol)


def test_position_encoding_backward_is_deterministic(cuda):
    from deepctr_b200 import engine as E
    from deepctr_b200.layers import PositionEncoding
    B, T, Ed = 8192, 50, 64
    rng = np.random.RandomState(0)
    x = torch.tensor(rng.normal(size=(B, T, Ed)).astype(np.float32), device=cuda)
    g = torch.tensor(rng.normal(size=(B, T, Ed)).astype(np.float32), device=cuda)
    grads = []
    for _ in range(2):
        E.clear_session()
        pe = PositionEncoding()
        v = E.Var(x, requires_grad=True)
        pe._maybe_build((None, T, Ed))
        pe.lookup_table.materialize()
        tape = E.Tape()
        with E.recording(tape):
            y = pe._invoke(v, False)
        y.requires_grad = True
        E.add_grad(y, g)
        tape.backward()
        grads.append(pe.lookup_table.grad.clone())
    assert torch.equal(grads[0], grads[1])
    want = g.double().sum(0) * Ed ** 0.5
    _close(grads[0], want, "d lookup_table", 1e-5)


# ---- the BST builder -------------------------------------------------------------------------------------------
def _bst_data(rng, n, T, vocab=(40, 12), dims=(8, 8)):
    from deepctr_b200.feature_column import SparseFeat, VarLenSparseFeat, DenseFeat
    cols = [SparseFeat('user', 20, embedding_dim=dims[0]), SparseFeat('gender', 2, embedding_dim=dims[0]),
            SparseFeat('item_id', vocab[0] + 1, embedding_dim=dims[0]),
            SparseFeat('cate_id', vocab[1] + 1, embedding_dim=dims[1]), DenseFeat('pay_score', 1)]
    cols += [VarLenSparseFeat(SparseFeat('hist_item_id', vocab[0] + 1, embedding_dim=dims[0], embedding_name='item_id'),
                              maxlen=T, length_name="seq_length"),
             VarLenSparseFeat(SparseFeat('hist_cate_id', vocab[1] + 1, embedding_dim=dims[1], embedding_name='cate_id'),
                              maxlen=T, length_name="seq_length")]
    ln = rng.randint(0, T + 1, size=n).astype(np.int32)
    ln[:3] = [0, 1, T]
    pos = np.arange(T)[None, :] < ln[:, None]
    x = {'user': rng.randint(0, 20, n).astype(np.int32), 'gender': rng.randint(0, 2, n).astype(np.int32),
         'item_id': rng.randint(1, vocab[0] + 1, n).astype(np.int32),
         'cate_id': rng.randint(1, vocab[1] + 1, n).astype(np.int32),
         'pay_score': rng.rand(n).astype(np.float32),
         'hist_item_id': (rng.randint(1, vocab[0] + 1, (n, T)) * pos).astype(np.int32),
         'hist_cate_id': (rng.randint(1, vocab[1] + 1, (n, T)) * pos).astype(np.int32),
         'seq_length': ln.reshape(n, 1)}
    y = (rng.rand(n) < 0.4).astype(np.float32)
    return cols, x, y


def _bst_train(graph, update, init=None, steps=5, **kw):
    from deepctr_b200 import engine as E, models as M
    from deepctr_b200.engine import SGD
    cols, x, y = _bst_data(np.random.RandomState(7), 256, 10)
    E.clear_session()
    model = M.BST(cols, ['item_id', 'cate_id'], att_head_num=4, l2_reg_embedding=0, seed=3, **kw)
    if init is None:
        H.randomize_weights(model, np.random.RandomState(1), std=0.2)
        init = [w.value() for w in model.weights]
    else:
        model.set_weights(init)
    model.compile(SGD(0.05), "binary_crossentropy", embedding_update=update, step_graph=graph)
    losses = [model.train_on_batch(x, y) for _ in range(steps)]
    return losses, {w.name: w.value() for w in model.weights}, model.replayed_launches, init


@pytest.mark.parametrize("kw", [dict(), dict(transformer_num=2, dnn_hidden_units=())], ids=["default", "two_layers"])
def test_bst_graph_replayed_step_equals_eager(cuda, kw):
    # (the 'sparse' embedding update adds duplicate ids' rows with fp32 atomics: runs differ by reordered sums)
    l_graph, w_graph, replayed, init = _bst_train("auto", "sparse", **kw)
    l_eager, w_eager, _, _ = _bst_train("off", "sparse", init=init, **kw)
    assert replayed > 0, "the training step was never replayed as a CUDA graph"
    assert np.all(np.isfinite(l_graph))
    np.testing.assert_allclose(l_graph, l_eager, rtol=1e-4, atol=1e-6)
    for k, v in w_eager.items():
        np.testing.assert_allclose(w_graph[k], v, rtol=1e-3, atol=1e-5 + 5e-4 * float(np.abs(v).max()), err_msg=k)


def test_bst_sparse_and_dense_embedding_updates_agree(cuda):
    # the 'sparse' update adds duplicate ids' rows with fp32 atomics, so the two runs differ by reordered sums
    l_s, w_s, _, init = _bst_train("off", "sparse", steps=2)
    l_d, w_d, _, _ = _bst_train("off", "dense", init=init, steps=2)
    np.testing.assert_allclose(l_s, l_d, rtol=1e-4, atol=1e-6)
    for k, v in w_d.items():
        np.testing.assert_allclose(w_s[k], v, rtol=1e-3, atol=1e-5 + 5e-4 * float(np.abs(v).max()), err_msg=k)


def test_bst_with_dropout_trains_eagerly(cuda):
    losses, _, replayed, _ = _bst_train("auto", "sparse", dnn_dropout=0.2)
    assert replayed == 0 and np.all(np.isfinite(losses))


def test_bst_c4_shaped_step(cuda):
    """B = 8192, T = 50, E = 64 (item 48 + category 16), 8 heads of 8: two training steps run, the loss is finite
    and moves."""
    from deepctr_b200 import engine as E, models as M
    from deepctr_b200.engine import SGD
    cols, x, y = _bst_data(np.random.RandomState(2), 8192, 50, vocab=(100000, 1000), dims=(48, 16))
    E.clear_session()
    model = M.BST(cols, ['item_id', 'cate_id'], att_head_num=8, l2_reg_embedding=0)
    model.compile(SGD(0.05), "binary_crossentropy", embedding_update="sparse")
    l0 = model.train_on_batch(x, y)
    l1 = model.train_on_batch(x, y)
    assert np.isfinite(l0) and np.isfinite(l1) and l0 != l1
