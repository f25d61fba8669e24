"""GPU: the Criteo fast-path embedding kernels - the uniform gather and its atomic scatter (embed.cu), the sorted
deterministic update (embed_sorted.cu), their row-sharded peer instantiations (SHARD = true) and the a2a shard
kernels (shard.cu) - called directly through deepctr_b200.kernels at the production shapes and at the edges, and
compared with torch restatements of the same operation that run on the device.

The sharded kernels take DEVICE arrays of shard pointers, so all the shards of a world of G ranks can live on one
device: the peer path and the a2a schedule are emulated in-process, exactly, with no second GPU.

Shapes: C2 (B = 65536, F = 26, V = 1M, dim 32, 13 dense columns, ldx 848), C3 (B = 32768, dim 16) and C5 per GPU
(B = 32768, F = 26, dim 128, V reduced to 100k per table).  Ids are uniform or Zipf(1.05) truncated to the
vocabulary (bench.py's IdSampler), int32 and int64, handed to the kernels as strided columns of one [B, F] matrix.

Bounds (U = 2^-24, the fp32 unit roundoff; a sum of n terms in any order, tree or sequence of depth d, is off by
at most d U sum|terms| <= (n - 1) U sum|terms| to first order):
- copies (x rows, dense columns, a2a rows, peer vs unsharded gathers): bit for bit;
- fm = 0.5 (sum_e S_e^2 - Q), S_e = sum_f x_fe, Q = sum x^2:
  0.5 ((2F + 11) U M + (5 ceil(F / RPI) + 6) U Q) + U |fm|, M = sum_e (sum_f |x_fe|)^2 >= Q.
  S_e has depth <= F (F U relative to sum_f |x_fe|, doubled by the square), sum_e S_e^2 adds 4 products per lane
  and a 5-level shuffle tree; each lane adds 4 products per feature it holds (ceil(F / RPI) of them) into q, then
  the same tree.  fm is a difference of two O(M) sums: the bound is absolute, never relative to fm;
- linear: F U sum_f |lin_f|;
- atomic SGD scatter (and the a2a / peer updates): for a touched row, (n_row + 4) U (|w0| + sum |scale| T1) +
  F U sum |scale dfm| sum_f |x_f|, T1 = |dx| + |dfm| (|S| + |x|) for an FM field, |dx| otherwise.  The first term
  is the sum of n_row + 1 terms (w0 and n_row gradient rows, red.add in any order) plus the three roundings of
  r = dx + dfm (S - x) and the scale; the second is the fp32 error of S (depth <= F) carried through dfm;
- sorted SGD: bit for bit against an fp32 restatement with one torch op per rounding;
- sorted Adagrad: acc bit for bit; w within 2U |w0| + 6U |q|, q = lr g / (sqrt(acc) + eps) (lr g may be an FMA,
  sqrt, + eps and / round once each, w - q once).
"""
import math

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
TINY = 1e-30
SENTINEL = 7.25
C2 = dict(B=65536, F=26, V=1000000, dim=32, nd=13, ldx=848)
C3 = dict(B=32768, F=26, V=1000000, dim=16, nd=13, ldx=432)
C5 = dict(B=32768, F=26, V=100000, dim=128, nd=13, ldx=3344)


def _kern():
    from deepctr_b200 import kernels as K, _lib as L
    return K, L


def _gen(dev, seed):
    g = torch.Generator(device=dev)
    g.manual_seed(seed)
    return g


def _normal(gen, shape, dev, std=1.0):
    return torch.empty(shape, dtype=torch.float32, device=dev).normal_(0.0, std, generator=gen)


def _ids(gen, B, F, V, dev, dist="uniform", dtype=torch.int32, bad=True):
    """[B, F] ids, uniform or Zipf(1.05) as bench.IdSampler draws them; `bad` puts ids -1, V, V + 7 (and, for
    int64, V + 2^33) at a few places."""
    if dist == "zipf":
        k = torch.arange(1, V + 1, dtype=torch.float64, device=dev)
        cdf = torch.cumsum(k.pow_(-1.05), 0)
        cdf /= cdf[-1].clone()
        ids = torch.searchsorted(cdf, torch.rand((B, F), generator=gen, dtype=torch.float64, device=dev))
        ids = ids.clamp_(max=V - 1)
    else:
        ids = torch.randint(0, V, (B, F), generator=gen, device=dev)
    if bad:
        ids[0, 0] = -1
        ids[B - 1, F - 1] = V
        ids[B // 2, F // 2] = V + 7
        if dtype == torch.int64:
            ids[B // 3, (F - 1) // 3] = V + (1 << 33)
    return ids.to(dtype)


def _valid(ids, V):
    i = ids.long()
    ok = (i >= 0) & (i < V)
    return ok, torch.where(ok, i, torch.zeros_like(i))


def _ref_rows(tabs, ids):
    """fp32 [B, F, dim] rows of the lookups, zero rows for ids outside the vocabulary."""
    F, V, dim = tabs.shape
    ok, safe = _valid(ids, V)
    rows = tabs[torch.arange(F, device=tabs.device)[None, :], safe]
    return rows.masked_fill_(~ok[..., None], 0.0), ok, safe


def _fm_sel(F, fm_mask, dev):
    return torch.tensor([(fm_mask >> f) & 1 == 1 for f in range(F)], dtype=torch.bool, device=dev)


def _within(got, want, bound, what):
    assert bool(torch.isfinite(got).all()), "%s: non-finite values" % what
    ratio = (got.double() - want).abs() / bound
    worst = float(ratio.max()) if ratio.numel() else 0.0
    assert worst <= 1.0, "%s: error %.3g times the bound" % (what, worst)


def _plan(K, tabs, ids, x, lins=None, dense=None, linear=None, fm=None, fm_mask=0, x_cols=0, vocab=None):
    F = ids.shape[1]
    feats = [K.make_feature(tabs[f], ids[:, f:f + 1], x, vocab=vocab) for f in range(F)]
    plan = K.UniformPlan(feats, None if lins is None else [lins[f] for f in range(F)], dense, x, linear, fm, fm_mask)
    plan.g.x_cols = x_cols
    return plan


def _check_fm(fm, rows, fm_mask, what):
    """fm against float64 within the absolute bound of the module docstring."""
    B, F, dim = rows.shape
    sel = _fm_sel(F, fm_mask, rows.device)
    r64 = rows.double() * sel[None, :, None]
    S = r64.sum(1)
    Q = (r64 * r64).sum((1, 2))
    want = 0.5 * ((S * S).sum(1) - Q)
    M = (r64.abs().sum(1) ** 2).sum(1)
    rpi = 32 // (dim // 4)
    bound = 0.5 * ((2 * F + 11) * U * M + (5 * math.ceil(F / rpi) + 6) * U * Q) + U * want.abs() + TINY
    _within(fm, want, bound, what)


def _check_linear(linear, lins, ok, safe, what):
    F = ok.shape[1]
    if lins is None:
        assert bool((linear == 0).all()), "%s: linear without lin tables must be 0" % what
        return
    v = lins[torch.arange(F, device=lins.device)[None, :], safe].double() * ok
    # F U sum |lin|: a sum of at most F nonzero terms
    _within(linear, v.sum(1), F * U * v.abs().sum(1) + TINY, what)


def _check_gather(x, fm, linear, tabs, lins, ids, dense, fm_mask, x_cols, what):
    B, F = ids.shape
    dim = tabs.shape[2]
    nd = dense.shape[1] if dense is not None else 0
    rows, ok, safe = _ref_rows(tabs, ids)
    c0 = F * dim
    assert torch.equal(x[:, :c0], rows.reshape(B, c0)), what + ": rows are not bit-exact copies"
    if nd:
        assert torch.equal(x[:, c0:c0 + nd], dense), what + ": dense columns are not bit-exact copies"
    xc = x_cols or x.shape[1]
    assert bool((x[:, c0 + nd:xc] == 0).all()), what + ": padding columns are not zero"
    if xc < x.shape[1]:
        assert bool((x[:, xc:] == SENTINEL).all()), what + ": columns at or beyond x_cols were written"
    if fm is not None:
        _check_fm(fm, rows, fm_mask, what + ": fm")
    if linear is not None:
        _check_linear(linear, lins, ok, safe, what + ": linear")
    return ok


# ================================================================================================
# A. uniform gather (world <= 1)
# ================================================================================================
def _run_gather(K, cuda, gen, B, F, V, dim, nd, ldx, dist, dtype, fm_mask, x_cols=0, with_fm=True, lin="tables",
                what=""):
    tabs = _normal(gen, (F, V, dim), cuda, 0.3)
    lins = _normal(gen, (F, V), cuda, 0.3) if lin == "tables" else None
    ids = _ids(gen, B, F, V, cuda, dist, dtype)
    dense = _normal(gen, (B, nd + 3), cuda)[:, 1:1 + nd] if nd else None     # a column window: dense_ld != nd
    x = torch.full((B, ldx), SENTINEL, device=cuda)
    fm = torch.empty((B,), device=cuda) if with_fm else None
    linear = torch.empty((B,), device=cuda) if lin is not None else None
    plan = _plan(K, tabs, ids, x, lins=lins, dense=dense, linear=linear, fm=fm, fm_mask=fm_mask, x_cols=x_cols)
    K.embed_oob_count(reset=True)
    K.embed_gather_uniform_fwd(plan, B)
    ok = _check_gather(x, fm, linear, tabs, lins, ids, dense, fm_mask, x_cols, what)
    assert K.embed_oob_count(reset=True) == int((~ok).sum()), what + ": out-of-range ids miscounted"


@pytest.mark.parametrize("shape,dist,dtype", [
    pytest.param(C2, "uniform", torch.int32, id="c2-uniform-i32"),
    pytest.param(C2, "zipf", torch.int64, id="c2-zipf-i64"),
    pytest.param(C3, "zipf", torch.int32, id="c3-zipf-i32"),
    pytest.param(C5, "uniform", torch.int64, id="c5-uniform-i64"),
])
def test_gather_production_shapes(cuda, shape, dist, dtype):
    K, L = _kern()
    s = shape
    _run_gather(K, cuda, _gen(cuda, 101), s["B"], s["F"], s["V"], s["dim"], s["nd"], s["ldx"], dist, dtype,
                (1 << s["F"]) - 1, what="gather %s" % dist)
    torch.cuda.empty_cache()


def _mask(kind, F):
    full = (1 << F) - 1
    if kind == "all":
        return full
    if kind == "holes":
        return full & ~((1 << 3) | (1 << (F // 2)) | 1)
    assert kind == "holes63" and F == 64
    return full & ~((1 << 3) | (1 << 40))            # bit 63 set


_EDGES = [pytest.param(F, 32, 300, 5, "all", 0, True, "tables", id="F%d" % F)
          for F in (1, 2, 27, 28, 29, 32, 33, 63)]
_EDGES += [pytest.param(64, 32, 300, 5, "holes63", 0, True, "tables", id="F64-bit63")]
_EDGES += [pytest.param(26, d, 300, 13, "holes", 0, True, "tables", id="dim%d" % d) for d in (4, 8, 16, 32, 64, 128)]
_EDGES += [
    pytest.param(26, 32, 1, 13, "all", 0, True, "tables", id="B1"),
    pytest.param(26, 128, 1, 0, "all", 0, True, "tables", id="B1-dim128"),
    pytest.param(26, 32, 5, 13, "holes", 0, True, "tables", id="B5"),
    pytest.param(40, 8, 300, 5, "holes", 1, True, "tables", id="xcols-lt-ldx"),
    pytest.param(26, 16, 300, 0, "all", -1, True, "tables", id="xcols-embeddings-only"),
    pytest.param(26, 32, 300, 13, "all", 0, False, "tables", id="fm-null"),
    pytest.param(26, 32, 300, 13, "all", 0, True, "null", id="lin-tables-null"),
    pytest.param(33, 64, 300, 3, "holes", 0, False, None, id="fm-and-linear-null"),
]


@pytest.mark.parametrize("F,dim,B,nd,mask,xc,with_fm,lin", _EDGES)
@pytest.mark.parametrize("dtype", [torch.int32, torch.int64], ids=["i32", "i64"])
def test_gather_edges(cuda, F, dim, B, nd, mask, xc, with_fm, lin, dtype):
    """F around the U*RPI pass and the lane / lane + 32 split, every dim, B below the grid's warp count, fm_mask
    holes and bit 63, x_cols < ldx (columns beyond keep a sentinel), and fm / linear / lin tables NULL."""
    K, L = _kern()
    ldx = (F * dim + nd + 3) // 4 * 4 + 8
    x_cols = 0
    if xc == 1:
        x_cols = F * dim + nd + 1                      # one zero column, the rest keeps the sentinel
    elif xc == -1:
        x_cols = F * dim                               # PNN's placement: the gather owns only the embeddings
    _run_gather(K, cuda, _gen(cuda, 7 * F + dim + B), B, F, 1000, dim, nd, ldx, "uniform", dtype,
                _mask(mask, F), x_cols=x_cols, with_fm=with_fm, lin=lin, what="gather F%d dim%d B%d" % (F, dim, B))


# ================================================================================================
# B. uniform scatter, atomic SGD (world <= 1)
# ================================================================================================
def _ref_update(ids, V, x, dx, dfm, dlin, fm_mask, scale, lin_scale, dim):
    """float64 update of the touched rows: (u = f * V + id, delta [nu, dim], bound terms, lin delta, lin terms,
    n_row).  Only the touched rows are formed (torch.unique + index_add_)."""
    B, F = ids.shape
    dev = x.device
    ok, safe = _valid(ids, V)
    sel = _fm_sel(F, fm_mask, dev)[None, :, None].double()
    xr = x[:, :F * dim].reshape(B, F, dim).double()
    r = dx[:, :F * dim].reshape(B, F, dim).double() if dx is not None else torch.zeros_like(xr)
    t1 = r.abs()
    t2 = torch.zeros_like(xr)
    if dfm is not None:
        S = (xr * sel).sum(1, keepdim=True)
        Sa = (xr.abs() * sel).sum(1, keepdim=True)
        d = dfm.double()[:, None, None]
        tmp = torch.sub(S, xr).mul_(d).mul_(sel)
        r += tmp
        torch.abs(xr, out=tmp).add_(S.abs()).mul_(d.abs()).mul_(sel)
        t1 += tmp
        del tmp
        t2 += (d.abs() * Sa) * sel
        del S, Sa
    del xr
    key = (torch.arange(F, device=dev)[None, :] * V + safe)[ok]
    u, inv = torch.unique(key, return_inverse=True)
    nu = u.numel()
    okf = ok.reshape(-1)

    def acc(v):
        return torch.zeros((nu,) + v.shape[2:], dtype=torch.float64, device=dev).index_add_(
            0, inv, v.reshape((B * F,) + v.shape[2:])[okf])
    delta = acc(r) * scale
    mag = acc(t1) * abs(scale)
    mag2 = acc(t2) * abs(scale)
    del r, t1, t2
    n = acc(torch.ones((B, F), dtype=torch.float64, device=dev))
    lv = dlin.double()[:, None].expand(B, F) if dlin is not None else torch.zeros((B, F), dtype=torch.float64,
                                                                                  device=dev)
    dl = acc(lv) * lin_scale
    dla = acc(lv.abs()) * abs(lin_scale)
    return u, delta, mag, mag2, dl, dla, n, F


def _check_update(tab_rows_new, w0u, lin_new, l0u, ref, what):
    u, delta, mag, mag2, dl, dla, n, F = ref
    bound = (n[:, None] + 4) * U * (w0u.double().abs() + mag) + F * U * mag2 + TINY
    _within(tab_rows_new.double() - w0u.double(), delta, bound, what + ": table rows")
    if lin_new is not None:
        lb = (n + 4) * U * (l0u.double().abs() + dla) + TINY
        _within(lin_new.double() - l0u.double(), dl, lb, what + ": lin rows")


def _rowsums(tabs):
    """float64 row sums of a [F, V, dim] table, one feature at a time (no float64 copy of the whole table)."""
    return torch.stack([tabs[f].sum(-1, dtype=torch.float64) for f in range(tabs.shape[0])])


def _restore_and_check_untouched(tabs, lins, u, w0u, l0u, rowsum0, linsum0, what):
    """Write the touched rows back: the whole table must then equal what it was (untouched rows unchanged)."""
    dim = tabs.shape[2]
    tabs.view(-1, dim)[u] = w0u
    assert torch.equal(_rowsums(tabs), rowsum0), what + ": an untouched row changed"
    if lins is not None:
        lins.view(-1)[u] = l0u
        assert torch.equal(lins, linsum0), what + ": an untouched lin row changed"


@pytest.mark.parametrize("case", [
    pytest.param(dict(dist="uniform", dtype=torch.int32, mask="all"), id="c2-uniform"),
    pytest.param(dict(dist="zipf", dtype=torch.int64, mask="all"), id="c2-zipf"),
    pytest.param(dict(dist="zipf", dtype=torch.int32, mask="holes", lin_scale=-0.125), id="c2-zipf-holes-linscale"),
    pytest.param(dict(dist="zipf", dtype=torch.int32, mask="all", no="dx"), id="c2-dx-null"),
    pytest.param(dict(dist="zipf", dtype=torch.int64, mask="holes", no="dfm"), id="c2-dfm-null"),
    pytest.param(dict(dist="uniform", dtype=torch.int32, mask="all", no="dlinear"), id="c2-dlinear-null"),
])
def test_scatter_atomic_sgd_c2(cuda, case):
    """b2ctr_embed_scatter_uniform_bwd at C2: every touched row against the float64 update, untouched rows and
    out-of-range ids left alone, the dense columns of dx never read (they hold NaN)."""
    K, L = _kern()
    s = C2
    B, F, V, dim, nd, ldx = s["B"], s["F"], s["V"], s["dim"], s["nd"], s["ldx"]
    gen = _gen(cuda, 202)
    fm_mask = _mask(case["mask"], F)
    tabs = _normal(gen, (F, V, dim), cuda, 0.3)
    lins = _normal(gen, (F, V), cuda, 0.3)
    ids = _ids(gen, B, F, V, cuda, case["dist"], case["dtype"])
    x = torch.full((B, ldx), SENTINEL, device=cuda)
    plan = _plan(K, tabs, ids, x, lins=lins, fm_mask=fm_mask)
    K.embed_gather_uniform_fwd(plan, B)
    K.embed_oob_count(reset=True)
    dx = _normal(gen, (B, ldx), cuda)
    dx[:, F * dim:] = float("nan")
    dfm = _normal(gen, (B,), cuda)
    dlin = _normal(gen, (B,), cuda)
    no = case.get("no")
    dx, dfm, dlin = (None if no == "dx" else dx), (None if no == "dfm" else dfm), (None if no == "dlinear" else dlin)
    scale, lin_scale = -0.05, case.get("lin_scale", -0.05)
    ref = _ref_update(ids, V, x, dx, dfm, dlin, fm_mask, scale, lin_scale, dim)
    u = ref[0]
    w0u, l0u = tabs.view(-1, dim)[u].clone(), lins.view(-1)[u].clone()
    rowsum0, lin0 = _rowsums(tabs), lins.clone()
    K.embed_scatter_uniform_bwd(plan, dx, dfm, dlin, scale, lin_scale, B)
    what = "scatter %s" % case
    _check_update(tabs.view(-1, dim)[u], w0u, lins.view(-1)[u], l0u, ref, what)
    _restore_and_check_untouched(tabs, lins, u, w0u, l0u, rowsum0, lin0, what)
    del tabs, lins, x, ref
    torch.cuda.empty_cache()


@pytest.mark.parametrize("dtype", [torch.int32, torch.int64], ids=["i32", "i64"])
def test_scatter_store_grads(cuda, dtype):
    """B2CTR_UNIFORM_STORE_GRADS (the a2a path: ids are a permutation of positions in a private row buffer): the
    stored rows equal, bit for bit, the atomic scatter of the same gradients into a zeroed buffer (0 + v = v),
    and the float64 gradient within the bound."""
    K, L = _kern()
    B, F, dim, ldx = 8192, 26, 32, 848
    gen = _gen(cuda, 303)
    n = B * F
    ids = torch.randperm(n, generator=gen, device=cuda).view(B, F).to(dtype)
    x = _normal(gen, (B, ldx), cuda, 0.3)
    dx, dfm, dlin = _normal(gen, (B, ldx), cuda), _normal(gen, (B,), cuda), _normal(gen, (B,), cuda)
    fm_mask = _mask("holes", F)
    out = {}
    for store in (True, False):
        rows = torch.full((n, dim), float("nan"), device=cuda) if store else torch.zeros((n, dim), device=cuda)
        glin = torch.full((n,), float("nan"), device=cuda) if store else torch.zeros((n,), device=cuda)
        plan = _plan(K, [rows] * F, ids, x, lins=[glin] * F, fm_mask=fm_mask)
        plan.g.flags = L.UNIFORM_STORE_GRADS if store else 0
        K.embed_scatter_uniform_bwd(plan, dx, dfm, dlin, 1.0, 1.0, B)
        out[store] = (rows, glin)
    assert torch.equal(out[True][0], out[False][0]), "stored rows differ from the atomic scatter into zeros"
    assert torch.equal(out[True][1], out[False][1]), "stored lin values differ from the atomic scatter into zeros"
    ref = _ref_update(ids, n, x, dx, dfm, dlin, fm_mask, 1.0, 1.0, dim)
    # every table view is the same buffer: fold the per-feature keys f * n + pos back onto pos
    u = ref[0] % n
    _check_update(out[True][0][u], torch.zeros((u.numel(), dim), device=cuda), out[True][1][u],
                  torch.zeros((u.numel(),), device=cuda), ref, "store grads")


# ================================================================================================
# C. sorted update
# ================================================================================================
def _sorted_want(stores, group, ids, x, dx, dfm, dlin, fm_mask, lr, adagrad=False, accs=None, laccs=None,
                 lstores=None, eps=1e-7):
    """fp32 restatement of b2ctr_embed_update_sorted: S by sequential adds over the FM fields, r = dx + dfm (S - x)
    one op per rounding, a stable sort by (table, id), per-run sums in ascending (b, f) order, one update per row.
    stores: [T, V, dim] tables (feature f reads stores[group[f]]).  Returns (u, new rows | (rows64, acc),
    new lin | ...) for the touched rows u (flat index into stores.view(-1, dim))."""
    B, F = ids.shape
    T, V, dim = stores.shape
    dev = x.device
    xr = x[:, :F * dim].reshape(B, F, dim)
    r = dx[:, :F * dim].reshape(B, F, dim).clone()
    sel = _fm_sel(F, fm_mask, dev)
    if dfm is not None:
        S = torch.zeros((B, dim), device=dev)
        for f in range(F):
            if (fm_mask >> f) & 1:
                S = S + xr[:, f]
        t = S[:, None, :] - xr
        t = t * dfm[:, None, None]
        r = torch.where(sel[None, :, None], r + t, r)
        del t, S
    ok, safe = _valid(ids, V)
    grp = torch.tensor(group, dtype=torch.int64, device=dev)
    key = (grp[None, :] * V + safe).reshape(-1)
    nidx = torch.nonzero(ok.reshape(-1)).squeeze(1)                 # lookups in ascending n = b * F + f
    ks, perm = torch.sort(key[nidx], stable=True)
    src = nidx[perm]
    u, counts = torch.unique_consecutive(ks, return_counts=True)
    starts = torch.cumsum(counts, 0) - counts
    order = torch.argsort(counts, descending=True, stable=True)
    u, cnt, st = u[order], counts[order], starts[order]
    asc = cnt.flip(0).cpu()
    nk = (asc.numel() - torch.searchsorted(asc, torch.arange(int(asc[-1]) + 1), right=True)).tolist()
    rf = r.reshape(B * F, dim)
    g = rf[src[st]].clone()                                         # 0 + r = r
    gl = dlin[src[st] // F].clone() if dlin is not None else None
    for k in range(1, len(nk)):                                     # position k inside the runs longer than k
        m = nk[k]
        e = src[st[:m] + k]
        g[:m] = g[:m] + rf[e]
        if gl is not None:
            gl[:m] = gl[:m] + dlin[e // F]
    lr_t = torch.tensor(lr, dtype=torch.float32, device=dev)
    w0 = stores.view(-1, dim)[u]
    l0 = lstores.view(-1)[u] if lstores is not None else None
    if not adagrad:
        w = w0 - g * lr_t
        lw = l0 - gl * lr_t if (gl is not None and l0 is not None) else l0
        return u, w, lw
    a = accs.view(-1, dim)[u] + g * g
    w64 = w0.double() - lr * g.double() / (a.double().sqrt() + eps)
    q = (lr * g.double() / (a.double().sqrt() + eps)).abs()
    res = (u, (w64, a, w0, q))
    if gl is not None and l0 is not None:
        la = laccs.view(-1)[u] + gl * gl
        lq = (lr * gl.double() / (la.double().sqrt() + eps))
        res = res + ((l0.double() - lq, la, l0, lq.abs()),)
    return res


def _sorted_call(K, stores, lstores, group, ids, x, dx, dfm, dlin, fm_mask, lr, opt=0, accs=None, laccs=None):
    B, F = ids.shape
    tabs = [stores[group[f]] for f in range(F)]
    lins = [lstores[group[f]] for f in range(F)] if lstores is not None else None
    plan = _plan(K, tabs, ids, x, lins=lins, fm_mask=fm_mask)
    acc = [accs[group[f]] for f in range(F)] if accs is not None else None
    lacc = [laccs[group[f]] for f in range(F)] if laccs is not None else None
    K.embed_update_sorted(plan, dx, dfm, dlin, opt, lr, lr, 1e-7, acc, lacc, B)


@pytest.mark.parametrize("dtype,mask", [(torch.int32, "all"), (torch.int64, "holes")], ids=["i32", "i64-holes"])
def test_sorted_sgd_c2_zipf_bit_exact(cuda, dtype, mask):
    """C2 with Zipf ids: runs thousands of lookups long, 1.7M keys (cub's multi-tile sort), ids -1 and V.
    Bit for bit against the fp32 restatement, and bit-identical on a second run."""
    K, L = _kern()
    s = C2
    B, F, V, dim, ldx = s["B"], s["F"], s["V"], s["dim"], s["ldx"]
    gen = _gen(cuda, 404)
    fm_mask = _mask(mask, F)
    tabs = _normal(gen, (F, V, dim), cuda, 0.3)
    lins = _normal(gen, (F, V), cuda, 0.3)
    ids = _ids(gen, B, F, V, cuda, "zipf", dtype)
    x = torch.full((B, ldx), SENTINEL, device=cuda)
    K.embed_gather_uniform_fwd(_plan(K, tabs, ids, x, fm_mask=fm_mask), B)
    K.embed_oob_count(reset=True)
    dx, dfm, dlin = _normal(gen, (B, ldx), cuda), _normal(gen, (B,), cuda), _normal(gen, (B,), cuda)
    lr = 0.05
    group = list(range(F))
    u, w_want, l_want = _sorted_want(tabs, group, ids, x, dx, dfm, dlin, fm_mask, lr, lstores=lins)
    assert int(torch.bincount(ids[:, 0].long().clamp(0, V - 1)).max()) > 1000       # long runs were reached
    w0u, l0u = tabs.view(-1, dim)[u].clone(), lins.view(-1)[u].clone()
    rowsum0, lin0 = _rowsums(tabs), lins.clone()
    got = []
    for rep in range(2):
        _sorted_call(K, tabs, lins, group, ids, x, dx, dfm, dlin, fm_mask, lr)
        got.append((tabs.view(-1, dim)[u].clone(), lins.view(-1)[u].clone()))
        _restore_and_check_untouched(tabs, lins, u, w0u, l0u, rowsum0, lin0, "sorted sgd rep %d" % rep)
    assert torch.equal(got[0][0], w_want), "sorted SGD rows are not bit-exact"
    assert torch.equal(got[0][1], l_want), "sorted SGD lin rows are not bit-exact"
    assert torch.equal(got[0][0], got[1][0]) and torch.equal(got[0][1], got[1][1]), "runs differ"
    del tabs, lins, x
    torch.cuda.empty_cache()


def _check_adagrad(stores, accs, lstores, laccs, want, what):
    dim = stores.shape[2]
    u, (w64, a, w0, q) = want[0], want[1]
    assert torch.equal(accs.view(-1, dim)[u], a), what + ": accumulators are not bit-exact"
    _within(stores.view(-1, dim)[u], w64, 2 * U * w0.double().abs() + 6 * U * q + TINY, what + ": rows")
    if len(want) > 2:
        lw64, la, l0, lq = want[2]
        assert torch.equal(laccs.view(-1)[u], la), what + ": lin accumulators are not bit-exact"
        _within(lstores.view(-1)[u], lw64, 2 * U * l0.double().abs() + 6 * U * lq + TINY, what + ": lin rows")


@pytest.mark.parametrize("dtype", [torch.int32, torch.int64], ids=["i32", "i64"])
def test_sorted_adagrad_zipf(cuda, dtype):
    """Keras' lazy Adagrad on the sorted path at B = 65536, F = 26, dim 32 and V = 20000 (it needs accumulators):
    acc bit for bit, w within the bound (lr g / (sqrt(acc) + eps) may contract)."""
    K, L = _kern()
    B, F, V, dim, ldx = 65536, 26, 20000, 32, 848
    gen = _gen(cuda, 505)
    fm_mask = _mask("holes", F)
    tabs = _normal(gen, (F, V, dim), cuda, 0.3)
    lins = _normal(gen, (F, V), cuda, 0.3)
    accs = torch.full_like(tabs, 0.1)
    laccs = torch.full_like(lins, 0.1)
    ids = _ids(gen, B, F, V, cuda, "zipf", dtype)
    x = torch.full((B, ldx), SENTINEL, device=cuda)
    K.embed_gather_uniform_fwd(_plan(K, tabs, ids, x, fm_mask=fm_mask), B)
    K.embed_oob_count(reset=True)
    dx, dfm, dlin = _normal(gen, (B, ldx), cuda), _normal(gen, (B,), cuda), _normal(gen, (B,), cuda)
    want = _sorted_want(tabs, list(range(F)), ids, x, dx, dfm, dlin, fm_mask, 0.1, adagrad=True, accs=accs,
                        laccs=laccs, lstores=lins)
    _sorted_call(K, tabs, lins, list(range(F)), ids, x, dx, dfm, dlin, fm_mask, 0.1, opt=1, accs=accs, laccs=laccs)
    _check_adagrad(tabs, accs, lins, laccs, want, "adagrad")


_SHARED = [0, 0, 1, 0, 2, 1]          # feature -> table: features 0, 1, 3 share table 0; 2 and 5 share table 1


@pytest.mark.parametrize("opt", ["sgd", "adagrad"])
@pytest.mark.parametrize("mask", ["all", "holes"])
def test_sorted_shared_tables(cuda, opt, mask):
    """Features that share one table (and its lin table and accumulators), with ids duplicated across them: each
    row gets ONE update, from the ordered sum over all of its lookups in ascending (b, f); bit-identical runs."""
    K, L = _kern()
    B, F, V, dim, T = 4099, len(_SHARED), 37, 16, 3
    ldx = F * dim + 4
    gen = _gen(cuda, 606)
    fm_mask = _mask(mask, F) if mask == "all" else 0b101101
    stores = _normal(gen, (T, V, dim), cuda, 0.3)
    lstores = _normal(gen, (T, V), cuda, 0.3)
    ids = _ids(gen, B, F, V, cuda, "zipf", torch.int32)
    ids[:, 1] = ids[:, 0]                                          # the same id in two features of one table
    ids[7, 1] = -1
    x = torch.full((B, ldx), SENTINEL, device=cuda)
    K.embed_gather_uniform_fwd(_plan(K, [stores[g] for g in _SHARED], ids, x, fm_mask=fm_mask), B)
    K.embed_oob_count(reset=True)
    dx, dfm, dlin = _normal(gen, (B, ldx), cuda), _normal(gen, (B,), cuda), _normal(gen, (B,), cuda)
    lr = 0.05
    s0, l0 = stores.clone(), lstores.clone()
    results = []
    for rep in range(2):
        stores.copy_(s0)
        lstores.copy_(l0)
        accs, laccs = (torch.full_like(stores, 0.1), torch.full_like(lstores, 0.1)) if opt == "adagrad" else (None, None)
        want = _sorted_want(stores, _SHARED, ids, x, dx, dfm, dlin, fm_mask, lr, adagrad=opt == "adagrad",
                            accs=accs, laccs=laccs, lstores=lstores)
        _sorted_call(K, stores, lstores, _SHARED, ids, x, dx, dfm, dlin, fm_mask, lr, opt=1 if opt == "adagrad" else 0,
                     accs=accs, laccs=laccs)
        results.append((stores.clone(), lstores.clone()))
        if opt == "sgd":
            u, w, lw = want
            got = stores.view(-1, dim)[u]
            assert torch.equal(got, w), "shared table: %d of %d touched rows differ, max |diff| %.3g" % (
                int((got != w).any(1).sum()), u.numel(), float((got - w).abs().max()))
            assert torch.equal(lstores.view(-1)[u], lw), "shared table: lin rows differ"
        else:
            _check_adagrad(stores, accs, lstores, laccs, want, "shared-table adagrad")
    assert torch.equal(results[0][0], results[1][0]) and torch.equal(results[0][1], results[1][1]), (
        "shared table: runs differ in %d elements" % int((results[0][0] != results[1][0]).sum()))


def test_sorted_shared_table_needs_shared_state(cuda):
    """Two features on one table but with different lin tables or accumulators: ValueError, nothing launched."""
    K, L = _kern()
    B, V, dim = 64, 11, 8
    tab = torch.zeros((V, dim), device=cuda)
    lin_a, lin_b = torch.zeros((V,), device=cuda), torch.zeros((V,), device=cuda)
    ids = torch.zeros((B, 2), dtype=torch.int32, device=cuda)
    x = torch.zeros((B, 2 * dim), device=cuda)
    dx, dlin = torch.zeros_like(x), torch.zeros((B,), device=cuda)
    plan = _plan(K, [tab, tab], ids, x, lins=[lin_a, lin_b])
    n0 = L.launch_count()
    with pytest.raises(ValueError, match="share a table"):
        K.embed_update_sorted(plan, dx, None, dlin, 0, 0.1, 0.1, 1e-7, None, None, B)
    plan = _plan(K, [tab, tab], ids, x, lins=[lin_a, lin_a])
    accs = [torch.zeros_like(tab), torch.zeros_like(tab)]
    with pytest.raises(ValueError, match="share a table"):
        K.embed_update_sorted(plan, dx, None, dlin, 1, 0.1, 0.1, 1e-7, accs, [lin_a, lin_a], B)
    assert L.launch_count() == n0


@pytest.mark.parametrize("opt_name", ["sgd", "adagrad"])
def test_deepfm_shared_embedding_name_sorted_training(cuda, opt_name):
    """Model level: a DeepFM whose first two single-valued SparseFeats share an embedding_name, trained with
    embedding_update='sparse_deterministic' SGD / row-wise Adagrad for 3 steps against the CPU oracle trained by
    torch.optim on dense gradients."""
    import b2_helpers as H
    from oracle import models as OM
    from oracle import ops as O
    from deepctr_b200 import engine as E, ops
    from deepctr_b200.engine import SGD, Adagrad
    from deepctr_b200.feature_column import SparseFeat, DenseFeat
    from deepctr_b200.models import DeepFM
    ops.set_gemm_precision("fp32")
    try:
        rng = np.random.RandomState(707)
        n, V = 96, 12
        cols = [SparseFeat("C0", V, 8, embedding_name="shared"), SparseFeat("C1", V, 8, embedding_name="shared")]
        cols += [SparseFeat("C%d" % i, 20 + i, 8) for i in range(2, 5)]
        cols += [DenseFeat("I%d" % i, 1) for i in range(3)]
        x = {"C0": rng.randint(0, V, size=n).astype(np.int32)}
        x["C1"] = np.where(rng.rand(n) < 0.5, x["C0"], rng.randint(0, V, size=n)).astype(np.int32)
        x.update({"C%d" % i: rng.randint(0, 20 + i, size=n).astype(np.int32) for i in range(2, 5)})
        x.update({"I%d" % i: rng.rand(n).astype(np.float32) for i in range(3)})
        y = (rng.rand(n) < 0.3).astype(np.float32)
        E.clear_session()
        model = DeepFM(cols, cols, dnn_hidden_units=(16, 8), l2_reg_linear=0, l2_reg_embedding=0)
        H.randomize_weights(model, rng)
        lr = 0.05
        model.compile(SGD(lr) if opt_name == "sgd" else Adagrad(lr), "binary_crossentropy",
                      embedding_update="sparse_deterministic" if opt_name == "sgd" else "sparse")
        assert model.planner.sorted_update
        W = H.oracle_weights(model, requires_grad=True)
        params = list(H.flat_params(W).values())
        topt = (torch.optim.SGD(params, lr=lr) if opt_name == "sgd" else
                torch.optim.Adagrad(params, lr=lr, initial_accumulator_value=0.1, eps=1e-7))
        for step in range(3):
            topt.zero_grad()
            logit, pred = OM.deepfm(x, cols, cols, W)
            loss = O.binary_crossentropy(y, pred)
            loss.backward()
            got = model.train_on_batch(x, y)
            assert abs(got - float(loss.detach())) < 2e-5 * max(1.0, abs(float(loss.detach()))), (step, got)
            topt.step()
        new = H.flat_params(H.oracle_weights(model))
        for name, p in H.flat_params(W).items():
            np.testing.assert_allclose(new[name].numpy(), p.detach().numpy(), rtol=2e-4, atol=2e-6, err_msg=name)
    finally:
        ops.set_gemm_precision("bf16x3")


# ================================================================================================
# D. row-sharded peer path (SHARD = true), a world of G ranks emulated on one GPU
# ================================================================================================
class _Shards(object):
    """Rank g's shard of table f is full[f][g::G] (local row r // G of global row r), each held in a buffer with
    zero guard rows on either side; ptrs is the device array of shard pointers at entry f * G + g.  Behind the
    shard the guard region is V / 2 rows for G > 2, so that a kernel that got the local row wrong (r // 2 instead
    of r // G) still reads and writes inside the allocation and fails the comparison instead of faulting."""

    def __init__(self, full, G):
        self.G = G
        V = full.shape[1]
        tail = (V + 1) // 2 if G > 2 else 1
        self.bufs, self.n = [], []
        ptrs = []
        for f in range(full.shape[0]):
            row = []
            for g in range(G):
                part = full[f][g::G]
                buf = torch.zeros((1 + part.shape[0] + tail,) + tuple(part.shape[1:]), device=full.device)
                buf[1:1 + part.shape[0]] = part
                row.append(buf)
                ptrs.append(buf[1:].data_ptr())
                if f == 0:
                    self.n.append(part.shape[0])
            self.bufs.append(row)
        self.ptrs = torch.tensor(ptrs, dtype=torch.int64, device=full.device)

    def assemble(self, like):
        out = torch.empty_like(like)
        for f, row in enumerate(self.bufs):
            for g, buf in enumerate(row):
                out[f][g::self.G] = buf[1:1 + self.n[g]]
        return out

    def guards_zero(self):
        return all(bool((b[0] == 0).all()) and bool((b[1 + self.n[g]:] == 0).all())
                   for row in self.bufs for g, b in enumerate(row))


_PEER = [pytest.param(G, d, 26, 1024, 4099, id="G%d-dim%d" % (G, d)) for G in (2, 4, 8)
         for d in (4, 8, 16, 32, 64, 128)]
_PEER += [pytest.param(4, 32, 64, 512, 4099, id="G4-dim32-F64"), pytest.param(8, 128, 64, 256, 4099, id="G8-dim128-F64"),
          pytest.param(2, 4, 64, 512, 4099, id="G2-dim4-F64"),
          pytest.param(2, 128, 26, 8192, 100000, id="c5-tables-G2")]


@pytest.mark.parametrize("G,dim,F,Br,V", _PEER)
def test_peer_sharded_gather_and_scatter(cuda, G, dim, F, Br, V):
    """Forward: every emulated rank's x / fm / linear equal the unsharded gather bit for bit (same arithmetic,
    only the load addresses differ).  Backward: the G ranks' scatters with scale -lr / G leave every shard equal
    to the float64 update of the unsharded table over the global batch; guard rows stay zero; out-of-range ids are
    zero rows, counted, and skipped."""
    K, L = _kern()
    gen = _gen(cuda, 808 + G + dim + F)
    full = _normal(gen, (F, V, dim), cuda, 0.3)
    lfull = _normal(gen, (F, V), cuda, 0.3)
    sh, lsh = _Shards(full, G), _Shards(lfull, G)
    dummy = torch.full((V, dim), float("nan"), device=cuda)      # feats[f].table is ignored when world > 1
    fm_mask = _mask("holes", F)
    ldx = F * dim + 4
    idss, xs = [], []
    for r in range(G):
        ids = _ids(gen, Br, F, V, cuda, "zipf" if r % 2 else "uniform", torch.int64 if r % 2 else torch.int32)
        want = [torch.full((Br, ldx), SENTINEL, device=cuda), torch.empty((Br,), device=cuda),
                torch.empty((Br,), device=cuda)]
        K.embed_gather_uniform_fwd(_plan(K, full, ids, want[0], lins=lfull, linear=want[2], fm=want[1],
                                         fm_mask=fm_mask), Br)
        n_bad_ref = K.embed_oob_count(reset=True)
        got = [torch.full((Br, ldx), SENTINEL, device=cuda), torch.empty((Br,), device=cuda),
               torch.empty((Br,), device=cuda)]
        plan = _plan(K, [dummy] * F, ids, got[0], linear=got[2], fm=got[1], fm_mask=fm_mask, vocab=V)
        plan.set_peers(G, sh.ptrs, lsh.ptrs)
        K.embed_gather_uniform_fwd(plan, Br)
        assert K.embed_oob_count(reset=True) == n_bad_ref == int((~_valid(ids, V)[0]).sum())
        for name, a, b in zip(("x", "fm", "linear"), got, want):
            assert torch.equal(a, b), "rank %d: sharded %s differs from the unsharded gather" % (r, name)
        idss.append(ids)
        xs.append(got[0])
    # backward: rank by rank, into the peer shards
    gen_b = _gen(cuda, 909)
    dxs = [_normal(gen_b, (Br, ldx), cuda) for _ in range(G)]
    dfms = [_normal(gen_b, (Br,), cuda) for _ in range(G)]
    dlins = [_normal(gen_b, (Br,), cuda) for _ in range(G)]
    lr = 0.5
    sc = -lr / G
    ids_all, x_all = torch.cat(idss), torch.cat(xs)
    ref = _ref_update(ids_all, V, x_all, torch.cat(dxs), torch.cat(dfms), torch.cat(dlins), fm_mask, sc, sc, dim)
    u = ref[0]
    w0u, l0u = full.view(-1, dim)[u].clone(), lfull.view(-1)[u].clone()
    for r in range(G):
        bplan = _plan(K, [dummy] * F, idss[r], xs[r], fm_mask=fm_mask, vocab=V)
        bplan.set_peers(G, sh.ptrs, lsh.ptrs)
        K.embed_scatter_uniform_bwd(bplan, dxs[r], dfms[r], dlins[r], sc, sc, Br)
    new, lnew = sh.assemble(full), lsh.assemble(lfull)
    assert sh.guards_zero() and lsh.guards_zero(), "a guard row around a shard was written"
    _check_update(new.view(-1, dim)[u], w0u, lnew.view(-1)[u], l0u, ref, "peer G%d dim%d F%d" % (G, dim, F))
    new.view(-1, dim)[u] = w0u
    lnew.view(-1)[u] = l0u
    assert torch.equal(new, full) and torch.equal(lnew, lfull), "a row outside the global batch changed"
    del full, lfull, sh, lsh, new, lnew, ref
    torch.cuda.empty_cache()


def test_peer_sharded_rejections(cuda):
    """ValueError and nothing launched for: G not a power of two, G > 1 without peer tables, STORE_GRADS with
    G > 1, and the sorted update with G > 1."""
    K, L = _kern()
    B, F, V, dim = 16, 3, 40, 8
    tabs = torch.zeros((F, V, dim), device=cuda)
    ids = torch.zeros((B, F), dtype=torch.int32, device=cuda)
    x = torch.zeros((B, F * dim), device=cuda)
    ptrs = torch.tensor([tabs[f].data_ptr() for f in range(F) for _ in range(4)], dtype=torch.int64, device=cuda)
    n0 = L.launch_count()
    plan = _plan(K, tabs, ids, x)
    plan.set_peers(3, ptrs, None)
    with pytest.raises(ValueError, match="power of two"):
        K.embed_gather_uniform_fwd(plan, B)
    plan = _plan(K, tabs, ids, x)
    plan.g.world = 2
    with pytest.raises(ValueError, match="peer_tables"):
        K.embed_gather_uniform_fwd(plan, B)
    plan = _plan(K, tabs, ids, x)
    plan.set_peers(2, ptrs, None)
    plan.g.flags = L.UNIFORM_STORE_GRADS
    with pytest.raises(ValueError, match="STORE_GRADS"):
        K.embed_scatter_uniform_bwd(plan, x, None, None, 1.0, 1.0, B)
    plan = _plan(K, tabs, ids, x)
    plan.set_peers(2, ptrs, None)
    with pytest.raises(ValueError, match="row-sharded"):
        K.embed_update_sorted(plan, x, None, None, 0, 0.1, 0.1, 1e-7, None, None, B)
    assert L.launch_count() == n0


# ================================================================================================
# E. a2a shard kernels and their schedule, a world of G ranks emulated on one GPU
# ================================================================================================
def _id_feats(K, ids, V, dummy):
    return [K.make_feature(dummy, ids[:, f:f + 1], dummy, vocab=V) for f in range(ids.shape[1])]


def _route(K, ids, V, G, dummy):
    """bucketize + fill for one rank, with the checks of both kernels.  -> counts, offsets, keys, pos"""
    B, F = ids.shape
    feats = _id_feats(K, ids, V, dummy)
    K.embed_oob_count(reset=True)
    counts, slot = K.shard_bucketize(feats, B, G)
    ok, safe = _valid(ids, V)
    assert K.embed_oob_count(reset=True) == int((~ok).sum()), "bucketize: out-of-range ids miscounted"
    own = (safe % G).reshape(-1)                                   # out-of-range ids are routed as id 0
    cnt = torch.bincount(own, minlength=G)
    assert torch.equal(counts.long(), cnt), "bucketize: counts"
    assert torch.equal(slot >> 32, own), "bucketize: owner"
    rank = slot & 0xffffffff
    # inside each owner the ranks are a permutation of [0, count)
    off = torch.cumsum(cnt, 0) - cnt
    n = B * F
    got = torch.sort(own * n + rank).values
    own_s = torch.sort(own).values
    want = own_s * n + torch.arange(n, device=ids.device) - off[own_s]      # owner o: o * n + [0, count_o)
    assert torch.equal(got, want), "bucketize: ranks inside an owner are not a permutation of [0, count)"
    keys, pos = K.shard_fill(feats, B, G, counts, slot)
    p = pos.long().reshape(-1)
    assert torch.equal(torch.sort(p).values, torch.arange(B * F, device=ids.device)), "fill: pos is not a permutation"
    assert bool(((p >= off[own]) & (p < off[own] + cnt[own])).all()), "fill: pos outside its owner's segment"
    fidx = torch.arange(F, device=ids.device)[None, :].expand(B, F).reshape(-1)
    assert torch.equal(keys[p], (fidx << 40) | (safe.reshape(-1) // G)), "fill: keys"
    return cnt, off, keys, pos


_A2A = [pytest.param(G, B, dt, id="G%d-B%d-%s" % (G, B, "i32" if dt == torch.int32 else "i64"))
        for G in (1, 2, 3, 4, 8, 64) for B, dt in ((50, torch.int32), (4096, torch.int64))]


@pytest.mark.parametrize("G,B,dtype", _A2A)
def test_a2a_bucketize_and_fill(cuda, G, B, dtype):
    """b2ctr_shard_bucketize / _fill at B*F below one 2048-item block and well above it, with out-of-range ids."""
    K, L = _kern()
    gen = _gen(cuda, 1001 + G + B)
    V = 5003
    ids = _ids(gen, B, 26, V, cuda, "zipf", dtype)
    _route(K, ids, V, G, torch.zeros((1, 4), device=cuda))


@pytest.mark.parametrize("dim", [4, 8, 16, 32, 64, 128])
def test_a2a_gather_and_scatter_rows(cuda, dim):
    """shard_gather_rows: exact copies, a NULL lin table gives 0 and lin_tables NULL gives no lin output.
    shard_scatter_rows: duplicate keys, lin_scale != scale, glin NULL; float64 within the bound."""
    K, L = _kern()
    gen = _gen(cuda, 1100 + dim)
    F, R, n = 5, 37, 3001
    tabs = _normal(gen, (F, R, dim), cuda)
    lins = _normal(gen, (F, R), cuda)
    f = torch.randint(0, F, (n,), generator=gen, device=cuda)
    row = torch.randint(0, R, (n,), generator=gen, device=cuda)
    keys = (f << 40) | row
    lin_list = [lins[i] for i in range(F)]
    lin_list[2] = None
    rows, lout = K.shard_gather_rows([tabs[i] for i in range(F)], lin_list, dim, keys, n)
    assert torch.equal(rows[:n], tabs[f, row]), "gather_rows: rows"
    assert torch.equal(lout[:n], torch.where(f == 2, torch.zeros_like(lout[:n]), lins[f, row])), "gather_rows: lin"
    rows2, lout2 = K.shard_gather_rows([tabs[i] for i in range(F)], None, dim, keys, n)
    assert lout2 is None and torch.equal(rows2[:n], rows[:n])
    g = _normal(gen, (n, dim), cuda)
    gl = _normal(gen, (n,), cuda)
    for glin, lin_scale in ((gl, -0.25), (None, -0.25)):
        t, lt = tabs.clone(), lins.clone()
        K.shard_scatter_rows([t[i] for i in range(F)], [lt[i] for i in range(F)], dim, keys, n, g, glin, -0.5,
                             lin_scale)
        key = f * R + row
        cnt = torch.zeros(F * R, dtype=torch.float64, device=cuda).index_add_(0, key, torch.ones_like(key,
                                                                              dtype=torch.float64))
        d = torch.zeros((F * R, dim), dtype=torch.float64, device=cuda).index_add_(0, key, g.double() * -0.5)
        m = torch.zeros((F * R, dim), dtype=torch.float64, device=cuda).index_add_(0, key, g.double().abs() * 0.5)
        w0 = tabs.view(-1, dim).double()
        # sum of cnt + 1 terms in any order, one rounding of the scale each: (cnt + 2) U (|w0| + sum|scale g|)
        _within(t.view(-1, dim).double() - w0, d, (cnt[:, None] + 2) * U * (w0.abs() + m) + TINY, "scatter_rows")
        if glin is None:
            assert torch.equal(lt, lins), "scatter_rows: lin tables changed without glin"
        else:
            dl = torch.zeros(F * R, dtype=torch.float64, device=cuda).index_add_(0, key, gl.double() * lin_scale)
            ml = torch.zeros(F * R, dtype=torch.float64, device=cuda).index_add_(0, key, gl.double().abs()
                                                                                  * abs(lin_scale))
            l0 = lins.view(-1).double()
            _within(lt.view(-1).double() - l0, dl, (cnt + 2) * U * (l0.abs() + ml) + TINY, "scatter_rows lin")


@pytest.mark.parametrize("G,dim,dtype", [(1, 32, torch.int32), (2, 32, torch.int64), (3, 16, torch.int32),
                                         (4, 128, torch.int64), (8, 4, torch.int32), (64, 8, torch.int64)])
def test_a2a_schedule(cuda, G, dim, dtype):
    """parallel.ShardedExchange for G in-process ranks, with slicing in place of all_to_all_single: route, fetch,
    the uniform gather over the returned rows with pos as ids (x / fm / linear equal to the unsharded gather bit
    for bit), the STORE_GRADS scatter into the gradient rows, push and shard_scatter_rows with -lr / G (every shard
    equal to the float64 global-batch update).  G = 3: the a2a transport needs no power of two."""
    K, L = _kern()
    gen = _gen(cuda, 1200 + G + dim)
    F, Br, V = 26, 512, 3001
    full = _normal(gen, (F, V, dim), cuda, 0.3)
    lfull = _normal(gen, (F, V), cuda, 0.3)
    shards = [[full[f][g::G].clone() for f in range(F)] for g in range(G)]
    lshards = [[lfull[f][g::G].clone() for f in range(F)] for g in range(G)]
    dummy = torch.zeros((1, 4), device=cuda)
    fm_mask = _mask("holes", F)
    ldx = F * dim + 16
    routes, idss = [], []
    for r in range(G):
        ids = _ids(gen, Br, F, V, cuda, "zipf" if r % 2 else "uniform", dtype, bad=False)
        idss.append(ids)
        routes.append(_route(K, ids, V, G, dummy))
    # keys to the owners: owner g receives the g-th segment of every rank, in rank order
    recv = [torch.cat([routes[r][2][int(routes[r][1][g]):int(routes[r][1][g] + routes[r][0][g])] for r in range(G)])
            for g in range(G)]
    served = [K.shard_gather_rows(shards[g], lshards[g], dim, recv[g], recv[g].numel()) for g in range(G)]
    xs, sends = [], []
    for r in range(G):
        cnt, off = routes[r][0], routes[r][1]
        parts, lparts = [], []
        for g in range(G):
            start = sum(int(routes[q][0][g]) for q in range(r))
            c = int(cnt[g])
            parts.append(served[g][0][start:start + c])
            lparts.append(served[g][1][start:start + c])
        back, blin = torch.cat(parts), torch.cat(lparts)
        pos = routes[r][3]
        want = [torch.full((Br, ldx), SENTINEL, device=cuda), torch.empty((Br,), device=cuda),
                torch.empty((Br,), device=cuda)]
        K.embed_gather_uniform_fwd(_plan(K, full, idss[r], want[0], lins=lfull, linear=want[2], fm=want[1],
                                         fm_mask=fm_mask), Br)
        got = [torch.full((Br, ldx), SENTINEL, device=cuda), torch.empty((Br,), device=cuda),
               torch.empty((Br,), device=cuda)]
        K.embed_gather_uniform_fwd(_plan(K, [back] * F, pos, got[0], lins=[blin] * F, linear=got[2], fm=got[1],
                                         fm_mask=fm_mask), Br)
        for name, a, b in zip(("x", "fm", "linear"), got, want):
            assert torch.equal(a, b), "rank %d: a2a %s differs from the unsharded gather" % (r, name)
        xs.append(got[0])
        sends.append(back.shape[0])
    gen_b = _gen(cuda, 1300)
    dxs = [_normal(gen_b, (Br, ldx), cuda) for _ in range(G)]
    dfms = [_normal(gen_b, (Br,), cuda) for _ in range(G)]
    dlins = [_normal(gen_b, (Br,), cuda) for _ in range(G)]
    grows, glins = [], []
    for r in range(G):
        gr = torch.empty((sends[r], dim), device=cuda)
        gl = torch.empty((sends[r],), device=cuda)
        bplan = _plan(K, [gr] * F, routes[r][3], xs[r], lins=[gl] * F, fm_mask=fm_mask)
        bplan.g.flags = L.UNIFORM_STORE_GRADS
        K.embed_scatter_uniform_bwd(bplan, dxs[r], dfms[r], dlins[r], 1.0, 1.0, Br)
        grows.append(gr)
        glins.append(gl)
    lr = 0.5
    sc = -lr / G
    for g in range(G):
        seg = [(int(routes[r][1][g]), int(routes[r][0][g])) for r in range(G)]
        g_recv = torch.cat([grows[r][o:o + c] for r, (o, c) in enumerate(seg)])
        gl_recv = torch.cat([glins[r][o:o + c] for r, (o, c) in enumerate(seg)])
        K.shard_scatter_rows(shards[g], lshards[g], dim, recv[g], recv[g].numel(), g_recv, gl_recv, sc, sc)
    new, lnew = torch.empty_like(full), torch.empty_like(lfull)
    for g in range(G):
        for f in range(F):
            new[f][g::G] = shards[g][f]
            lnew[f][g::G] = lshards[g][f]
    ref = _ref_update(torch.cat(idss), V, torch.cat(xs), torch.cat(dxs), torch.cat(dfms), torch.cat(dlins), fm_mask,
                      sc, sc, dim)
    u = ref[0]
    # the gradient rows are stored at scale 1 (exact) and scaled by their owner: the same roundings as the fused
    # scatter, so B's bound
    _check_update(new.view(-1, dim)[u], full.view(-1, dim)[u], lnew.view(-1)[u], lfull.view(-1)[u], ref,
                  "a2a G%d" % G)
    new.view(-1, dim)[u] = full.view(-1, dim)[u]
    lnew.view(-1)[u] = lfull.view(-1)[u]
    assert torch.equal(new, full) and torch.equal(lnew, lfull), "a row outside the global batch changed"


def test_a2a_rejections(cuda):
    """ValueError and nothing launched for a dim outside {4, ..., 128}, a misaligned table, nfeat > 64 and
    world > 64."""
    K, L = _kern()
    keys = torch.zeros((4,), dtype=torch.int64, device=cuda)
    buf = torch.zeros((64 * 260 + 1,), device=cuda)
    ok_tab = buf[:64 * 256].view(64, 256)
    n0 = L.launch_count()
    for dim in (2, 12, 256):
        with pytest.raises(ValueError, match="dim"):
            K.shard_gather_rows([ok_tab[:, :dim].contiguous()], None, dim, keys, 4)
        with pytest.raises(ValueError, match="dim"):
            K.shard_scatter_rows([ok_tab], None, dim, keys, 4, torch.zeros((4, 256), device=cuda), None, 1.0, 1.0)
    bad = buf[1:1 + 64 * 32].view(64, 32)                         # 4-byte offset: not 16-byte aligned
    with pytest.raises(ValueError, match="misaligned"):
        K.shard_gather_rows([bad], None, 32, keys, 4)
    with pytest.raises(ValueError, match="misaligned"):
        K.shard_scatter_rows([bad], None, 32, keys, 4, torch.zeros((4, 32), device=cuda), None, 1.0, 1.0)
    dummy = torch.zeros((1, 4), device=cuda)
    ids = torch.zeros((8, 65), dtype=torch.int32, device=cuda)
    counts = torch.zeros((65,), dtype=torch.int32, device=cuda)
    slot = torch.zeros((8 * 65,), dtype=torch.int64, device=cuda)
    feats = _id_feats(K, ids, 10, dummy)
    arr = (L.Feature * 65)(*feats)
    with pytest.raises(ValueError, match="nfeat"):
        K._lib_call("shard_bucketize", arr, 65, 8, 2, K.ptr(counts), K.ptr(slot), K.stream())
    with pytest.raises(ValueError, match="nfeat"):
        K._lib_call("shard_fill", arr, 65, 8, 2, K.ptr(counts), K.ptr(slot), K.ptr(slot), K.ptr(counts), K.stream())
    with pytest.raises(ValueError, match="bad tables"):
        K.shard_gather_rows([dummy] * 65, None, 4, keys, 4)
    with pytest.raises(ValueError, match="bad arguments"):
        K._lib_call("shard_bucketize", arr, 8, 8, 65, K.ptr(counts), K.ptr(slot), K.stream())
    with pytest.raises(ValueError, match="bad arguments"):
        K._lib_call("shard_fill", arr, 8, 8, 65, K.ptr(counts), K.ptr(slot), K.ptr(slot), K.ptr(counts), K.stream())
    assert L.launch_count() == n0
