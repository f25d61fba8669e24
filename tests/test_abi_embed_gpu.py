"""GPU parity: embedding gather / scatter / hash kernels through the C-ABI vs the CPU oracle.

Bit-exact for rows, ids, masks and unweighted pooled sums (SURVEY.md section 8c); fp32 tolerance
(stated per test) where softmax / exp is involved.
"""
import numpy as np
import pytest
import torch

from oracle import ops as O
from oracle import farmhash

pytestmark = pytest.mark.gpu


def _kern():
    from deepctr_b200 import kernels as K, _lib as L
    return K, L


def _mk_tables(rng, nf, vocab, dim, dev, std=0.05):
    tabs = [torch.tensor(rng.normal(0, std, size=(vocab, dim)).astype(np.float32)) for _ in range(nf)]
    return tabs, [t.to(dev) for t in tabs]


@pytest.mark.parametrize("dim", [1, 3, 4, 8, 32, 64, 130])
@pytest.mark.parametrize("dtype", [torch.int32, torch.int64])
def test_single_lookup_bit_exact(cuda, dim, dtype):
    K, L = _kern()
    rng = np.random.RandomState(0)
    B, F, V = 257, 5, 101
    host, dev = _mk_tables(rng, F, V, dim, cuda)
    idx = torch.tensor(rng.randint(0, V, size=(B, F)), dtype=dtype)
    idx_d = idx.to(cuda)
    ld = F * dim + 3
    out = torch.full((B, ld), -7.0, device=cuda)
    feats = [K.make_feature(dev[f], idx_d[:, f], out, out_col=f * dim, out_ld=ld) for f in range(F)]
    K.embed_gather_fwd(feats, B)
    got = out.cpu()
    for f in range(F):
        want = O.embedding_lookup(host[f], idx[:, f])[:, 0, :]
        assert torch.equal(got[:, f * dim:(f + 1) * dim], want)
    assert torch.all(got[:, F * dim:] == -7.0)  # untouched padding


@pytest.mark.parametrize("mode", ["sum", "mean", "max"])
@pytest.mark.parametrize("maskmode", ["length", "zero"])
@pytest.mark.parametrize("dim", [4, 6, 32, 130])
def test_pooled_bag_bit_exact(cuda, mode, maskmode, dim):
    """bags of 9 and of 50 positions; dim 130 takes the scalar path with several lane passes"""
    K, L = _kern()
    rng = np.random.RandomState(1)
    B, V = 131, 50
    host, dev = _mk_tables(rng, 1, V, dim, cuda, std=1.0)
    for T in (9, 50):
        lens = rng.randint(0, T + 1, size=B)
        lens[0], lens[1] = 0, T  # empty and full bags
        idx = rng.randint(1, V, size=(B, T))
        for b in range(B):
            idx[b, lens[b]:] = 0
        idx_t = torch.tensor(idx, dtype=torch.int32)
        seq = O.embedding_lookup(host[0], idx_t)
        if maskmode == "length":
            want = O.sequence_pooling(seq, mode, lengths=torch.tensor(lens))
            mask_mode, length = L.MASK_LENGTH, torch.tensor(lens, dtype=torch.int32, device=cuda)
        else:
            want = O.sequence_pooling(seq, mode, mask=idx_t != 0)
            mask_mode, length = L.MASK_ZERO_ID, None
        out = torch.empty((B, dim), device=cuda)
        f = K.make_feature(dev[0], idx_t.to(cuda), out, maxlen=T, pool=L.POOL_BY_NAME[mode],
                           mask_mode=mask_mode, length=length)
        K.embed_gather_fwd([f], B)
        assert torch.equal(out.cpu(), want[:, 0, :]), "pooled segment results must be bit-exact (T = %d)" % T


@pytest.mark.parametrize("norm", [True, False])
def test_weighted_bag(cuda, norm):
    K, L = _kern()
    rng = np.random.RandomState(2)
    B, T, V, dim = 64, 7, 40, 8
    host, dev = _mk_tables(rng, 1, V, dim, cuda, std=1.0)
    lens = rng.randint(1, T + 1, size=B)
    idx = rng.randint(1, V, size=(B, T))
    w = rng.rand(B, T).astype(np.float32)
    idx_t = torch.tensor(idx, dtype=torch.int64)
    seq = O.embedding_lookup(host[0], idx_t)
    ws = O.weighted_sequence(seq, torch.tensor(w), norm, lengths=torch.tensor(lens))
    want = O.sequence_pooling(ws, "sum", lengths=torch.tensor(lens))
    out = torch.empty((B, dim), device=cuda)
    f = K.make_feature(dev[0], idx_t.to(cuda), out, maxlen=T, pool=L.POOL_SUM, mask_mode=L.MASK_LENGTH,
                       length=torch.tensor(lens, dtype=torch.int32, device=cuda),
                       weight=torch.tensor(w, device=cuda),
                       weight_mode=L.WEIGHT_SOFTMAX if norm else L.WEIGHT_RAW)
    K.embed_gather_fwd([f], B)
    # softmax uses expf on both sides: fp32 tolerance 1e-6 relative (raw weights: exact products)
    torch.testing.assert_close(out.cpu(), want[:, 0, :], rtol=2e-6, atol=1e-7)


def test_sequence_emit_and_scatter(cuda):
    """POOL_NONE with maxlen=T emits the [B,T,E] key sequence (DIN); scatter routes grads back."""
    K, L = _kern()
    rng = np.random.RandomState(3)
    B, T, V, dim = 33, 5, 20, 16
    host, dev = _mk_tables(rng, 1, V, dim, cuda)
    idx = torch.tensor(rng.randint(0, V, size=(B, T)), dtype=torch.int32)
    out = torch.empty((B, T * dim), device=cuda)
    f = K.make_feature(dev[0], idx.to(cuda), out, maxlen=T)
    K.embed_gather_fwd([f], B)
    assert torch.equal(out.cpu().reshape(B, T, dim), O.embedding_lookup(host[0], idx))
    # scatter: dense gradient into a zeroed table
    g = torch.tensor(rng.normal(size=(B, T * dim)).astype(np.float32))
    gtab = torch.zeros((V, dim), device=cuda)
    fb = K.make_feature(gtab, idx.to(cuda), g.to(cuda), maxlen=T)
    K.embed_scatter_add([fb], B, 1.0)
    want = torch.zeros(V, dim).index_add_(0, idx.reshape(-1).long(), g.reshape(B * T, dim))
    torch.testing.assert_close(gtab.cpu(), want, rtol=1e-5, atol=1e-6)


NEG_PAD32 = float(np.float32(-4294967295.0))   # the softmax padding -2^32 + 1, which is -2^32 in fp32


def _bag64(tab64, ids, valid, mode, weight_mode=None, w=None):
    """float64 restatement of a pooled (optionally weighted) bag, sequence.py:76-106 and :155-183.  The max-pool mask
    x - 1e9 is computed in fp32 as the reference does (every masked |x| < 32 then ties at -1e9); its gradient is 1."""
    seq = tab64[torch.as_tensor(ids, dtype=torch.int64)]                           # [B, T, E]
    v = torch.as_tensor(valid)
    if weight_mode is not None:
        w64 = torch.as_tensor(w).double()
        if weight_mode == "softmax":
            wt = torch.softmax(torch.where(v, w64, torch.full_like(w64, NEG_PAD32)), dim=1)
        else:
            wt = torch.where(v, w64, torch.zeros_like(w64))
        seq = seq * wt[:, :, None]
    v3 = v[:, :, None]
    if mode == "max":
        s32 = seq.detach().float()
        hist = seq + (torch.where(v3, s32, s32 - 1e9).double() - seq).detach()
        return hist.amax(dim=1)
    out = (seq * v3).sum(dim=1)
    if mode == "mean":
        out = out / (v.sum(dim=1, keepdim=True).double() + 1e-8)
    return out


@pytest.mark.parametrize("mode", ["sum", "mean", "max"])
def test_pooled_scatter_matches_autograd(cuda, mode):
    """table gradient of pooled bags against float64 autograd: length and zero-id masks, a hashed feature, raw and
    softmax position weights, and a dim that is not a multiple of 4 (the scalar path)"""
    K, L = _kern()
    rng = np.random.RandomState(4)
    B, T, V = 50, 6, 30
    # (mask mode, hashed, weight mode, dim)
    cases = [("length", False, None, 8), ("zero", False, None, 8), ("zero", True, None, 6),
             ("length", False, "raw", 8), ("length", False, "softmax", 6), ("zero", True, "softmax", 8),
             ("zero", False, "raw", 6)]
    for maskmode, hashed, weight_mode, dim in cases:
        what = "%s mask, hashed=%s, weights %s, dim %d" % (maskmode, hashed, weight_mode, dim)
        host, dev = _mk_tables(rng, 1, V, dim, cuda, std=1.0)
        lens = rng.randint(0, T + 1, size=B)
        lens[0] = 0
        if hashed:
            raw = rng.randint(1, 10 ** 6, size=(B, T))
            raw[rng.rand(B, T) < 0.3] = 0                       # padding ids hash to bucket 0 and are masked
            raw[0] = 0
            ids = O.hash_layer(raw, V, mask_zero=True)
            idx = torch.tensor(raw, dtype=torch.int64)
        else:
            ids = rng.randint(0 if maskmode == "zero" else 1, V, size=(B, T))
            ids[0] = 0
            idx = torch.tensor(ids, dtype=torch.int32)
        valid = np.arange(T)[None, :] < lens[:, None] if maskmode == "length" else ids != 0
        w = rng.normal(size=(B, T)).astype(np.float32)
        tab = host[0].double().requires_grad_(True)
        pooled = _bag64(tab, ids, valid, mode, weight_mode, w)
        g = torch.tensor(rng.normal(size=(B, dim)).astype(np.float32))
        (pooled * g.double()).sum().backward()
        gtab = torch.zeros((V, dim), device=cuda)
        # max pooling re-reads the forward rows (src_table) to find the arg-max positions
        f = K.make_feature(gtab, idx.to(cuda), g.to(cuda), maxlen=T, pool=L.POOL_BY_NAME[mode],
                           mask_mode=L.MASK_LENGTH if maskmode == "length" else L.MASK_ZERO_ID,
                           length=torch.tensor(lens, dtype=torch.int32, device=cuda) if maskmode == "length" else None,
                           hash_mode=L.HASH_FARM_MASK_ZERO if hashed else L.HASH_NONE,
                           weight=torch.tensor(w, device=cuda) if weight_mode else None,
                           weight_mode={None: L.WEIGHT_NONE, "raw": L.WEIGHT_RAW, "softmax": L.WEIGHT_SOFTMAX}[weight_mode],
                           src_table=dev[0])
        K.embed_scatter_add([f], B, 1.0)
        # atomics add a row's contributions in any order: fp32 tolerance against float64
        torch.testing.assert_close(gtab.cpu().double(), tab.grad, rtol=1e-5, atol=1e-6, msg=what)


def test_mixed_features_one_launch(cuda):
    """~70 features of dims 3 / 8 / 64 / 130 in one gather and one scatter call (two 64-descriptor launches, the
    sub-warp width set by the widest feature): every pool mode, hashed and plain, int32 and int64 ids, each
    feature's ids (and lengths) a column window of one packed id buffer, weights a column window of a wider float
    buffer, outputs at out_col of a row wider than the features.  Unweighted results are bit-exact against the
    oracle; weighted ones and the scatter (atomics) are compared with float64."""
    K, L = _kern()
    rng = np.random.RandomState(21)
    B, V, nf = 301, 23, 70
    dims = [3, 8, 64, 130]
    pools = ["none", "sum", "mean", "max"]
    spec = []                                   # (dim, pool, T, hashed, int64, mask, weight)
    for i in range(nf):
        pool = pools[(i // 4) % 4]
        T = 1 if (pool == "none" and i % 3 == 0) else 2 + i % 6
        mask = "none" if pool == "none" else ("zero" if i % 3 == 0 else "length")
        weight = None if pool == "none" else [None, "raw", "softmax"][(i // 16) % 3]
        spec.append((dims[i % 4], pool, T, i % 3 == 0, i % 2 == 1, mask, weight))
    # packed id buffers (int32 also holds the lengths) and the weight buffer, each feature a column window
    n32 = n64 = 0
    cols = []                                   # (first id column, length column or None)
    for dim, pool, T, hashed, i64, mask, weight in spec:
        if i64:
            ic, n64 = n64, n64 + T
        else:
            ic, n32 = n32, n32 + T
        lc = None
        if mask == "length":
            lc, n32 = n32, n32 + 1
        cols.append((ic, lc))
    ids32 = np.zeros((B, n32 + 3), dtype=np.int32)
    ids64 = np.zeros((B, n64 + 3), dtype=np.int64)
    wcols = sum(T for _, _, T, *_ in spec)
    wbuf = rng.normal(size=(B, wcols + 5)).astype(np.float32)
    widths = [T * dim if pool == "none" else dim for dim, pool, T, *_ in spec]
    ld = sum(widths) + 7
    per = []                                    # reference inputs per feature
    wc = 0
    for (dim, pool, T, hashed, i64, mask, weight), (ic, lc) in zip(spec, cols):
        buf = ids64 if i64 else ids32
        raw = rng.randint(1, 10 ** 6 if hashed else V, size=(B, T))
        lens = rng.randint(0, T + 1, size=B)
        lens[0] = 0
        if mask == "zero":
            raw[rng.rand(B, T) < 0.3] = 0
            raw[0] = 0
        buf[:, ic:ic + T] = raw
        if lc is not None:
            ids32[:, lc] = lens
        ids = O.hash_layer(raw, V, mask_zero=True) if hashed else raw
        valid = (ids != 0) if mask == "zero" else (np.arange(T)[None, :] < lens[:, None]) if mask == "length" \
            else np.ones((B, T), dtype=bool)
        per.append((ids, valid, wc))
        wc += T
    host, dev = [], []
    for dim, *_ in spec:
        h, d = _mk_tables(rng, 1, V, dim, cuda, std=1.0)
        host.append(h[0])
        dev.append(d[0])
    i32_d, i64_d = torch.tensor(ids32, device=cuda), torch.tensor(ids64, device=cuda)
    w_d = torch.tensor(wbuf, device=cuda)
    out = torch.full((B, ld), -3.0, device=cuda)

    def feats(tables, target, src=None):
        fs, oc = [], 0
        for k, ((dim, pool, T, hashed, i64, mask, weight), (ic, lc), (_, _, wc0)) in enumerate(zip(spec, cols, per)):
            ib = i64_d if i64 else i32_d
            fs.append(K.make_feature(
                tables[k], ib[:, ic:ic + T], target, out_col=oc, out_ld=ld, maxlen=T,
                pool=L.POOL_NONE if pool == "none" else L.POOL_BY_NAME[pool],
                mask_mode={"none": L.MASK_NONE, "zero": L.MASK_ZERO_ID, "length": L.MASK_LENGTH}[mask],
                length=i32_d[:, lc] if lc is not None else None,
                weight=w_d[:, wc0:wc0 + T] if weight else None,
                weight_mode={None: L.WEIGHT_NONE, "raw": L.WEIGHT_RAW, "softmax": L.WEIGHT_SOFTMAX}[weight],
                hash_mode=L.HASH_FARM_MASK_ZERO if hashed else L.HASH_NONE,
                src_table=src[k] if src is not None else None))
            oc += widths[k]
        return fs

    K.embed_gather_fwd(feats(dev, out), B)
    got = out.cpu()
    assert torch.all(got[:, ld - 7:] == -3.0)                       # columns behind the last feature
    gout = torch.tensor(rng.normal(size=(B, ld)).astype(np.float32))
    tabs64 = [h.double().requires_grad_(True) for h in host]
    loss = 0
    oc = 0
    for k, (dim, pool, T, hashed, i64, mask, weight) in enumerate(spec):
        ids, valid, wc0 = per[k]
        seg = got[:, oc:oc + widths[k]]
        what = "feature %d (dim %d, %s, T %d, hashed %s, weights %s)" % (k, dim, pool, T, hashed, weight)
        idt = torch.tensor(ids, dtype=torch.int64)
        if pool == "none":
            assert torch.equal(seg, O.embedding_lookup(host[k], idt).reshape(B, T * dim)), what
            ref = tabs64[k][idt].reshape(B, T * dim)
        else:
            w = wbuf[:, wc0:wc0 + T]
            ref = _bag64(tabs64[k], ids, valid, pool, weight, w)
            if weight is None:
                want = O.sequence_pooling(O.embedding_lookup(host[k], idt), pool, mask=torch.tensor(valid))
                assert torch.equal(seg, want[:, 0, :]), what + ": unweighted pooling must be bit-exact"
            else:
                # a sum of at most 7 weighted rows of magnitude < 5: fp32 error well below 1e-5
                torch.testing.assert_close(seg.double(), ref.detach(), rtol=1e-5, atol=1e-5, msg=what)
        loss = loss + (ref * gout[:, oc:oc + widths[k]].double()).sum()
        oc += widths[k]
    loss.backward()
    grads = [torch.zeros_like(d) for d in dev]
    K.embed_scatter_add(feats(grads, gout.to(cuda), src=dev), B, 1.0)
    # each table row receives up to B*T/V ~ 90 contributions, added by atomics in any order: normwise fp32 tolerance
    for k, (dim, pool, T, hashed, i64, mask, weight) in enumerate(spec):
        ref = tabs64[k].grad
        err = float((grads[k].cpu().double() - ref).abs().max()) / float(ref.abs().max())
        assert err < 4e-6, "scatter of feature %d (dim %d, %s, weights %s): error %.3g" % (k, dim, pool, weight, err)


@pytest.mark.parametrize("dim", [4, 8, 16, 32, 64, 128])
@pytest.mark.parametrize("F,ndense", [(26, 13), (3, 0), (40, 5)])
def test_uniform_gather_fwd_bwd(cuda, dim, F, ndense):
    K, L = _kern()
    rng = np.random.RandomState(5)
    B, V = 300, 97
    host, dev = _mk_tables(rng, F, V, dim, cuda, std=0.3)
    lin_h = [torch.tensor(rng.normal(size=(V,)).astype(np.float32)) for _ in range(F)]
    lin_d = [t.to(cuda) for t in lin_h]
    idx = torch.tensor(rng.randint(0, V, size=(B, F)), dtype=torch.int32)
    idx_d = idx.to(cuda)
    dense = torch.tensor(rng.rand(B, max(ndense, 1)).astype(np.float32))[:, :ndense]
    ldx = (F * dim + ndense + 3) // 4 * 4 + 4
    x = torch.full((B, ldx), 9.0, device=cuda)
    linear = torch.empty((B,), device=cuda)
    fm = torch.empty((B,), device=cuda)
    feats = [K.make_feature(dev[f], idx_d[:, f], x) for f in range(F)]
    fm_mask = (1 << F) - 1 if F != 40 else ((1 << F) - 1) & ~0b1010
    dense_d = dense.to(cuda).contiguous() if ndense else None
    plan = K.UniformPlan(feats, lin_d, dense_d, x, linear, fm, fm_mask)
    K.embed_gather_uniform_fwd(plan, B)
    # oracle
    tabs = [t.clone().requires_grad_(True) for t in host]
    lins = [t.clone().requires_grad_(True) for t in lin_h]
    embs = [O.embedding_lookup(tabs[f], idx[:, f]) for f in range(F)]
    xe = torch.cat(embs, dim=1)
    sel = [f for f in range(F) if (fm_mask >> f) & 1]
    fm_want = O.fm(xe[:, sel, :])[:, 0]
    lin_want = sum(lins[f][idx[:, f].long()] for f in range(F))
    got = x.cpu()
    assert torch.equal(got[:, :F * dim], xe.reshape(B, F * dim).detach())       # rows: pure copy
    if ndense:
        assert torch.equal(got[:, F * dim:F * dim + ndense], dense)
    assert torch.all(got[:, F * dim + ndense:] == 0)                           # K padding is zero
    # FM is a difference of two O(sum x^2) terms: fp32 tolerance is relative to that magnitude
    mag = (xe[:, sel, :].detach().double() ** 2).sum(dim=(1, 2)) * len(sel)
    fm64 = O.fm(xe[:, sel, :].detach().double())[:, 0]
    assert ((fm.cpu().double() - fm64).abs() <= 2e-6 * mag + 1e-6).all()
    torch.testing.assert_close(linear.cpu(), lin_want.detach(), rtol=1e-5, atol=1e-5)
    # backward: dx, dfm, dlinear -> table deltas
    dx = torch.tensor(rng.normal(size=(B, ldx)).astype(np.float32))
    dfm = torch.tensor(rng.normal(size=(B,)).astype(np.float32))
    dlin = torch.tensor(rng.normal(size=(B,)).astype(np.float32))
    loss = (xe.reshape(B, -1) * dx[:, :F * dim]).sum() + (fm_want * dfm).sum() + (lin_want * dlin).sum()
    loss.backward()
    before = [t.clone() for t in dev]
    lbefore = [t.clone() for t in lin_d]
    lr = 0.5
    K.embed_scatter_uniform_bwd(plan, dx.to(cuda), dfm.to(cuda), dlin.to(cuda), -lr, -lr, B)
    for f in range(F):
        torch.testing.assert_close((dev[f] - before[f]).cpu(), -lr * tabs[f].grad, rtol=2e-4, atol=2e-5)
        torch.testing.assert_close((lin_d[f] - lbefore[f]).cpu(), -lr * lins[f].grad, rtol=2e-4, atol=2e-5)


def test_hash64_matches_oracle(cuda):
    K, L = _kern()
    rng = np.random.RandomState(6)
    ids = np.concatenate([np.arange(0, 200), rng.randint(0, 2 ** 31 - 1, size=500),
                          -rng.randint(1, 10 ** 6, size=50), [2 ** 31 - 1, 10 ** 9, 99999999]])
    for nb, mz in [(1000, False), (1000, True), (7, True), (1, False)]:
        want = O.hash_layer(ids, nb, mz)
        got = K.hash64(torch.tensor(ids, dtype=torch.int64, device=cuda), nb, mz).cpu().numpy()
        assert np.array_equal(got, want)
        got32 = K.hash64(torch.tensor(ids, dtype=torch.int32, device=cuda), nb, mz).cpu().numpy()
        assert np.array_equal(got32, want)
    big = np.array([2 ** 62 + 12345, -2 ** 63, 2 ** 63 - 1, 10 ** 18], dtype=np.int64)  # 19 and 20 chars
    got = K.hash64(torch.tensor(big, device=cuda), 10 ** 6, False).cpu().numpy()
    assert np.array_equal(got, O.hash_layer(big, 10 ** 6, False))


def test_hashed_lookup_in_kernel(cuda):
    K, L = _kern()
    rng = np.random.RandomState(7)
    B, T, V, dim = 40, 4, 64, 8
    host, dev = _mk_tables(rng, 1, V, dim, cuda)
    raw = rng.randint(0, 10 ** 6, size=(B, T))
    raw[:, -1] = 0  # padded tail
    hid = O.hash_layer(raw, V, mask_zero=True)
    seq = O.embedding_lookup(host[0], torch.tensor(hid))
    want = O.sequence_pooling(seq, "mean", mask=torch.tensor(hid) != 0)
    out = torch.empty((B, dim), device=cuda)
    f = K.make_feature(dev[0], torch.tensor(raw, dtype=torch.int64, device=cuda), out, maxlen=T,
                       pool=L.POOL_MEAN, mask_mode=L.MASK_ZERO_ID, hash_mode=L.HASH_FARM_MASK_ZERO)
    K.embed_gather_fwd([f], B)
    assert torch.equal(out.cpu(), want[:, 0, :])


def test_init_normal_statistics(cuda):
    K, L = _kern()
    t = torch.empty((1 << 20) + 3, device=cuda)
    K.init_normal(t, 0.0, 1e-4, 2020)
    h = t.cpu().double()
    assert abs(h.mean().item()) < 1e-6
    assert abs(h.std().item() / 1e-4 - 1.0) < 5e-3
    t2 = torch.empty_like(t)
    K.init_normal(t2, 0.0, 1e-4, 2020)
    assert torch.equal(t, t2)  # counter-based: reproducible


def test_invalid_arguments_raise_value_error(cuda):
    K, L = _kern()
    tab = torch.zeros((4, 4), device=cuda)
    out = torch.zeros((2, 4), device=cuda)
    f = K.make_feature(tab, torch.zeros(2, dtype=torch.int32, device=cuda), out, pool=7)
    with pytest.raises(ValueError):
        K.embed_gather_fwd([f], 2)


# ---- ids outside [0, vocab): zero rows, no out-of-bounds access in either direction, counted ----------
def test_out_of_range_ids_generic(cuda):
    K, L = _kern()
    rng = np.random.RandomState(11)
    B, T, V, dim = 64, 5, 37, 8
    host, dev = _mk_tables(rng, 1, V, dim, cuda, std=1.0)
    K.embed_oob_count(reset=True)
    idx = rng.randint(0, V, size=(B, T))
    idx[3, 1], idx[7, 0], idx[9, 4] = -1, V, 10 ** 9
    bad = (idx < 0) | (idx >= V)
    idx_t = torch.tensor(idx, dtype=torch.int32)
    out = torch.full((B, T * dim), 5.0, device=cuda)
    K.embed_gather_fwd([K.make_feature(dev[0], idx_t.to(cuda), out, maxlen=T)], B)
    want = host[0][torch.tensor(np.where(bad, 0, idx))].clone()
    want[torch.tensor(bad)] = 0.0
    assert torch.equal(out.cpu().reshape(B, T, dim), want)
    assert K.embed_oob_count(reset=True) == int(bad.sum())
    assert K.embed_oob_count(reset=True) == 0
    # pooled sum: an out-of-range id contributes a zero row
    pooled = torch.empty((B, dim), device=cuda)
    K.embed_gather_fwd([K.make_feature(dev[0], idx_t.to(cuda), pooled, maxlen=T, pool=L.POOL_SUM)], B)
    acc = torch.zeros(B, dim)
    for t in range(T):
        acc = acc + want[:, t, :]
    assert torch.equal(pooled.cpu(), acc)
    assert K.embed_oob_count(reset=True) == int(bad.sum())
    # scatter: guard rows around the table stay untouched, valid rows are updated
    guard = torch.zeros((V + 2, dim), device=cuda)
    tab = guard[1:V + 1]
    g = torch.ones((B, T * dim), device=cuda)
    K.embed_scatter_add([K.make_feature(tab, idx_t.to(cuda), g, maxlen=T)], B, 1.0)
    gh = guard.cpu()
    assert torch.all(gh[0] == 0) and torch.all(gh[V + 1] == 0)
    counts = np.bincount(idx[~bad].reshape(-1), minlength=V).astype(np.float32)
    assert torch.equal(gh[1:V + 1, 0], torch.tensor(counts))


@pytest.mark.parametrize("dim", [8, 32])
def test_out_of_range_ids_uniform(cuda, dim):
    K, L = _kern()
    rng = np.random.RandomState(12)
    B, F, V = 96, 6, 41
    host, dev = _mk_tables(rng, F, V, dim, cuda, std=0.5)
    lin_d = [torch.tensor(rng.normal(size=(V,)).astype(np.float32)).to(cuda) for _ in range(F)]
    idx = rng.randint(0, V, size=(B, F))
    idx[0, 0], idx[5, 3], idx[95, 5] = -7, V, V + 100
    bad = (idx < 0) | (idx >= V)
    idx_d = torch.tensor(idx, dtype=torch.int32).to(cuda)
    ldx = F * dim
    x = torch.full((B, ldx), 3.0, device=cuda)
    linear = torch.empty((B,), device=cuda)
    fm = torch.empty((B,), device=cuda)
    feats = [K.make_feature(dev[f], idx_d[:, f], x) for f in range(F)]
    plan = K.UniformPlan(feats, lin_d, None, x, linear, fm, (1 << F) - 1)
    K.embed_oob_count(reset=True)
    K.embed_gather_uniform_fwd(plan, B)
    got = x.cpu().reshape(B, F, dim)
    safe = np.where(bad, 0, idx)
    for f in range(F):
        want = host[f][torch.tensor(safe[:, f])].clone()
        want[torch.tensor(bad[:, f])] = 0.0
        assert torch.equal(got[:, f, :], want)
    lin_want = sum(torch.where(torch.tensor(bad[:, f]), torch.zeros(B), lin_d[f].cpu()[torch.tensor(safe[:, f])])
                   for f in range(F))
    torch.testing.assert_close(linear.cpu(), lin_want, rtol=1e-5, atol=1e-5)
    assert K.embed_oob_count(reset=True) == int(bad.sum())
    # backward into guarded copies of the tables
    guards = [torch.zeros((V + 2, dim), device=cuda) for _ in range(F)]
    lguards = [torch.zeros((V + 2,), device=cuda) for _ in range(F)]
    feats_b = [K.make_feature(guards[f][1:V + 1], idx_d[:, f], x) for f in range(F)]
    bplan = K.UniformPlan(feats_b, [lg[1:V + 1] for lg in lguards], None, x, None, None, (1 << F) - 1)
    dx = torch.ones((B, ldx), device=cuda)
    dlin = torch.ones((B,), device=cuda)
    K.embed_scatter_uniform_bwd(bplan, dx, None, dlin, 1.0, 1.0, B)
    for f in range(F):
        gh, lh = guards[f].cpu(), lguards[f].cpu()
        assert torch.all(gh[0] == 0) and torch.all(gh[V + 1] == 0) and lh[0] == 0 and lh[V + 1] == 0
        counts = np.bincount(idx[~bad[:, f], f], minlength=V).astype(np.float32)
        assert torch.equal(gh[1:V + 1, 0], torch.tensor(counts))
        assert torch.equal(lh[1:V + 1], torch.tensor(counts))


def test_model_raises_on_out_of_range_ids(cuda):
    """host mirror of TF-CPU's InvalidArgument (SURVEY.md App. A.1): predict / train_on_batch raise ValueError."""
    import b2_helpers as H
    from deepctr_b200.models import DeepFM
    rng = np.random.RandomState(13)
    cols, x, y = H.criteo_like(rng, 64)
    model = DeepFM(cols, cols, dnn_hidden_units=(8,))
    model.compile("sgd", "binary_crossentropy")
    assert model.predict(x, batch_size=64).shape == (64, 1)
    x["C0"] = x["C0"].copy()
    x["C0"][5] = -1
    with pytest.raises(ValueError, match="outside"):
        model.predict(x, batch_size=64)
    with pytest.raises(ValueError, match="outside"):
        model.train_on_batch(x, y)
    x["C0"][5] = 0
    model.train_on_batch(x, y)          # the counter was reset: clean data passes again
