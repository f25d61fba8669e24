"""GPU: the generic embedding gather and scatter, max pooling's per-position shares, the two mask kernels, the row
pack and FarmHash exactly, at their template, chunk and grid boundaries, with NaN in every padding.

Operands are exact.  Table rows are integers in [-8, 8] times 2^-2, raw weights integers in [-4, 4] times 2^-1,
gradients integers times 2^-1, and the update scale (the fused SGD's -lr) is -2^-3, so every term of every result
is a multiple of 2^-6.  Each check first asserts, from the data, that the sum of |terms| of each result stays below
2^24 of those units; every fp32 sum, red.add in any order included, is then exact, and gathers and scatters must
equal a float64 restatement bit for bit.  Where a kernel rounds once (a mean's division, a softmax weight 1/T) the
restatement rounds the same IEEE operation in fp32.  Three operations are made exact by their data:

* mean pooling: g is |L_b| times an integer, so g * scale / (L + 1e-8) is exact (L + 1e-8 == L in fp32 for |L| >= 1);
* max pooling: cnt, the number of positions attaining the max of (b, e), comes from the forward values and g is
  cnt times an integer;
* softmax weights: every valid weight is its row's maximum or at least 128 below it, with 1, 2 or 4 maxima, so the
  weights are 1/n or 0.  A row with no valid position weighs every position 1/T (one fp32 rounding); max pooling
  then ties all T positions at -1e9, and such rows get g = 0 unless T is a power of two.

The reference's fp32 masking constants are kept: x - 1e9 for a masked max position (every masked |x| < 32 then
ties at -1e9) and -2^32 for a masked softmax position.

Padding is poisoned and nothing outside a window may change: outputs and shares are windows of buffers filled
with a NaN that carries a payload; ids, lengths and weights are column windows of wider buffers whose other
columns and rows past the batch hold out-of-range ids (-1, vocab, 2^30, 2^31 / INT32_MIN), huge lengths and NaN
weights (a masked position's own weight is NaN too: the kernels must not use it).  b2ctr_embed_oob_count must
equal exactly the out-of-range ids the reference visits, so a stray read of a neighbouring id is counted.  Table
rows no id references are NaN for gathers and must keep their bits through scatters.

* every sub-warp width and vector path: float4 dims 4 / 8 / 12 / 16 / 32 / 64 / 68 / 128 / 132 / 256 (G 1, 2, 4
  with an idle lane, 4, 8, 16, 32 with an idle lane, 32, 32 with a partial second pass, 32 with two passes),
  scalar dims 1 / 2 / 3 / 5 / 31 / 33 / 65 / 130, dims % 4 == 0 forced onto the scalar path by out_col or out_ld,
  and narrow features in a launch whose G a wide one sets;
* every pool (none / sum / mean / max) x mask (none / zero id / length) x weight (none / raw / softmax), hashing
  none / farm / farm with mask_zero, int32 and int64 ids, T 1 / 3 / 4 / 5 / 50 / 200; empty and fully masked bags,
  lengths below 0 and above T, duplicate ids within a bag and across samples;
* tasks B * nfeat at the grid cap 1056 * 256 / G minus one, at it, plus one and past twice it for G 1, 8, 32, and
  nfeat 63 / 64 / 65 / 128 across the 64-descriptor chunk;
* the POOL_NONE scatter's all-zero-row skip: zero rows next to nonzero ones inside a warp, rows whose only nonzero
  is in the last lane or the second pass, rows of -0.0;
* the C4 shape: DIN's query gather and [8192, 50, 64] key gather from a 100,001-row table with Zipf ids, and the
  flat 409,600-row key scatter with half the gradients zero;
* max pooling under the fused update: b2ctr_embed_scatter_add refuses a max-pooled feature whose src_table is
  missing or is the table it updates; b2ctr_embed_max_pool_shares writes the shares at the forward rows and the
  POOL_NONE scatter applies them in place; a DeepFM with a max-pooled VarLen feature trained two SGD steps with
  embedding_update 'sparse' and 'dense' ends with bit-identical tables, and one step of an ONN with a max-pooled
  field-aware bag moves its tables by -lr x the dense gradient;
* a src_table that is not 16-byte aligned takes the scalar path;
* b2ctr_mask_from_len and b2ctr_mask_nonzero_and (first and AND modes, int32 / int64 ids nonzero only in their high
  half), n across the 270,336-thread cap, bytes past n unchanged;
* b2ctr_pack_rows with 1 / 2 / 63 / 64 blocks of widths 1, odd and wide, across the grid cap, ld_dst > total;
* b2ctr_hash64 and in-kernel hashing against oracle/farmhash.py at every decimal length 1-20, both signs, int32
  (INT32_MIN hashes as "-2147483648") and int64, num_buckets 1, 2 (mask_zero), a power of two and an odd value
  near 2^63.
"""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import farmhash

pytestmark = pytest.mark.gpu

NUM_SMS = 132
THREAD_CAP = NUM_SMS * 8 * 256           # grid_for(n, 256, 8): 1056 CTAs of 256 threads
NAN_BITS = 0x7fc00321                     # a quiet NaN with a payload
EXTRA = 3                                 # rows past the batch in every buffer
BIG_LEN = 1 << 30                         # the lengths around a length window
SCALE = -0.125                            # the fused SGD's -lr
UNIT = 2.0 ** -6                          # every scatter term is a multiple of this
NEG_PAD = -4294967296.0                   # -2^32 + 1 in fp32
INT32_MIN = -(1 << 31)
POOLS = ("none", "sum", "mean", "max")
MASKS = ("none", "zero", "length")
WEIGHTS = ("none", "raw", "softmax")
HASHES = ("none", "farm", "farm_mz")


def _kern():
    from deepctr_b200 import kernels as K, _lib as L
    return K, L


def _nan(shape, dev):
    return torch.full(tuple(shape), NAN_BITS, dtype=torch.int32, device=dev).view(torch.float32)


def _bits(t):
    return t.contiguous().view(torch.int32)


def _same(got, want, what):
    """fp32 ``got`` equals the float64 ``want`` (NaN never equals)."""
    g = got.double()
    bad = ~(g == want)
    n = int(bad.sum())
    if n:
        idx = tuple(int(i) for i in bad.nonzero()[0])
        raise AssertionError("%s: %d of %d entries differ, first at %s: got %r, want %r"
                             % (what, n, bad.numel(), idx, float(g[idx]), float(want[idx])))


def _fits(bound, what, unit=UNIT):
    top = float(bound.max()) if bound.numel() else 0.0
    assert top < 2.0 ** 24 * unit, "%s: the operands leave the exact range (%g)" % (what, top)


def _on_grid(terms, what, unit=UNIT):
    q = terms / unit
    assert bool((q == torch.round(q)).all()), "%s: a term is not a multiple of %g" % (what, unit)


def _f32(x):
    return x.to(torch.float32)


# ------------------------------------------------------------------------------------------------ features
class Spec:
    """One feature of a launch.  ``odd_col``: its out_col is not a multiple of 4."""

    def __init__(self, dim, T=1, pool="none", mask="none", weight="none", hash="none", i64=False, V=29,
                 odd_col=False, oob=True, table=None):
        self.dim, self.T, self.pool, self.mask, self.weight, self.hash = dim, T, pool, mask, weight, hash
        self.i64, self.V, self.odd_col, self.oob, self.table = i64, V, odd_col, oob, table

    @property
    def width(self):
        return self.T * self.dim if self.pool == "none" else self.dim

    def __repr__(self):
        return "dim %d T %d %s/%s/%s/%s %s" % (self.dim, self.T, self.pool, self.mask, self.weight, self.hash,
                                              "i64" if self.i64 else "i32")


def _hash(raw, V, mz):
    """oracle/farmhash.py on the distinct raw ids."""
    u, inv = np.unique(raw, return_inverse=True)
    h = np.array([farmhash.hash_bucket(int(v), V, mz) for v in u], dtype=np.int64)
    return h[inv].reshape(raw.shape)


def _zipf(rng, vocab, shape, low=0):
    """bench.py's IdSampler('zipf'): Zipf(1.05) truncated to the vocabulary."""
    w = 1.0 / np.arange(1, vocab + 1, dtype=np.float64) ** 1.05
    cdf = np.cumsum(w)
    cdf /= cdf[-1]
    r = np.searchsorted(cdf, rng.rand(*shape)).astype(np.int64)
    return np.minimum(r + low, vocab - 1)


class Launch:
    """Inputs, tables and output windows of one multi-feature launch, with a float64 reference of each feature."""

    def __init__(self, specs, B, seed, dev, ld_pad=5, ids=None, lens=None):
        K, L = _kern()
        self.specs, self.B, self.dev = specs, B, dev
        rng = np.random.RandomState(seed)
        self.rng = rng
        # ---- column layout: one poison column between windows, 2 after the last -------------------------------
        c32 = c64 = cl = cw = 0
        oc = 0
        self.lay = []
        for sp in specs:
            if sp.i64:
                ic, c64 = c64, c64 + sp.T + 1
            else:
                ic, c32 = c32, c32 + sp.T + 1
            lc = None
            if sp.mask == "length":
                lc, cl = cl, cl + 2
            wc = None
            if sp.weight != "none":
                wc, cw = cw, cw + sp.T + 1
            col = oc + (1 if sp.odd_col else 0)
            oc = (col + sp.width + 4) // 4 * 4
            self.lay.append((ic, lc, wc, col))
        self.ld = oc + ld_pad
        rows = B + EXTRA
        # ---- poison ----------------------------------------------------------------------------------------------
        p64 = np.array([-1, 1 << 30, 1 << 31, -(1 << 40)], dtype=np.int64)
        p32 = np.array([-1, 1 << 30, INT32_MIN, (1 << 31) - 1], dtype=np.int64)
        ids32 = p32[rng.randint(0, 4, size=(rows, c32 + 2))].astype(np.int32)
        ids64 = p64[rng.randint(0, 4, size=(rows, c64 + 2))]
        lenb = np.where(rng.rand(rows, cl + 2) < 0.5, BIG_LEN, -BIG_LEN).astype(np.int32)
        wb = np.full((rows, cw + 2), np.nan, dtype=np.float32)
        self.per = []
        self.n_oob = 0
        for k, (sp, (ic, lc, wc, col)) in enumerate(zip(specs, self.lay)):
            T, V = sp.T, sp.V
            # raw ids
            given = ids is not None and k in ids
            if given:
                raw = ids[k]
            elif sp.hash != "none":
                digits = rng.randint(1, 19, size=(B, T))
                raw = (rng.randint(0, 10 ** 9, size=(B, T)).astype(np.int64) * 10 ** 9
                       + rng.randint(0, 10 ** 9, size=(B, T))) % (10 ** digits)
                raw *= np.where(rng.rand(B, T) < 0.3, -1, 1)
                if not sp.i64:
                    raw = raw.astype(np.int32)   # wraps: every int32, INT32_MIN included
                    raw[0, 0] = INT32_MIN
            else:
                raw = rng.randint(0, V, size=(B, T)).astype(np.int64)
                # duplicate ids within a bag and across samples
                raw[:, T // 2:] = np.where(rng.rand(B, T - T // 2) < 0.3, raw[:, :1], raw[:, T // 2:])
                if B > 3:
                    raw[3] = raw[2]
                if sp.oob:
                    bad = rng.rand(B, T) < 0.03
                    far = (1 << 31) - 1 if not sp.i64 else 1 << 31
                    raw[bad] = np.array([-1, V, far])[rng.randint(0, 3, size=int(bad.sum()))]
            if not given and (sp.mask == "zero" or sp.hash == "farm_mz"):
                raw = np.where(rng.rand(B, T) < 0.3, 0, raw)
                raw[0] = 0                                           # an empty bag
            raw = np.asarray(raw, dtype=np.int64)
            if sp.i64:
                ids64[:B, ic:ic + T] = raw
                ids64[:, ic + T] = V                                 # the vocab right behind the window
            else:
                ids32[:B, ic:ic + T] = raw.astype(np.int32)
                ids32[:, ic + T] = V
            post = raw if sp.hash == "none" else _hash(raw, V, sp.hash == "farm_mz")
            # validity and lengths
            ln = None
            if sp.mask == "length":
                if lens is not None and k in lens:
                    ln = lens[k]
                else:
                    ln = rng.randint(-3, T + 4, size=B).astype(np.int32)
                    ln[:min(B, 4)] = [0, T, -2, T + 3][:min(B, 4)]
                lenb[:B, lc] = ln
                valid = np.arange(T)[None, :] < ln[:, None]
            elif sp.mask == "zero":
                valid = post != 0
            else:
                valid = np.ones((B, T), dtype=bool)
            if not given and B > 1 and sp.mask == "zero" and sp.hash == "none":
                valid[1] = False                                     # all positions masked
                post[1] = 0
                raw[1] = 0
                (ids64 if sp.i64 else ids32)[1, ic:ic + T] = 0
            # weights (a masked position's weight is NaN: it must not be used)
            w = None
            if sp.weight == "raw":
                w = (rng.randint(-4, 5, size=(B, T)) * 0.5).astype(np.float32)
            elif sp.weight == "softmax":
                nv = valid.sum(1)
                cap = np.where(nv >= 4, 4, np.where(nv >= 2, 2, 1))
                nw = np.minimum(np.array([1, 2, 4])[rng.randint(0, 3, size=B)], cap)
                key = rng.rand(B, T)
                key[~valid] = 2.0
                rank = np.argsort(np.argsort(key, 1), 1)
                win = (rank < nw[:, None]) & valid
                off = rng.randint(-40, 41, size=(B, 1)) * 0.125
                w = np.where(win, off, off - 128.0 * rng.randint(1, 5, size=(B, T))).astype(np.float32)
            if w is not None:
                w[~valid] = np.nan
                wb[:B, wc:wc + T] = w
            ok = (post >= 0) & (post < V)
            need = valid | (sp.pool in ("none", "max"))
            self.n_oob += int((need & ~ok).sum())
            self.per.append(dict(raw=raw, post=post, valid=valid, ok=ok, ln=ln, w=w))
        self.ids32 = torch.tensor(ids32, device=dev)
        self.ids64 = torch.tensor(ids64, device=dev)
        self.lenb = torch.tensor(lenb, device=dev)
        self.wb = torch.tensor(wb, device=dev)
        # ---- tables: referenced rows finite, every other row NaN ------------------------------------------------
        self.tables = []
        for k, sp in enumerate(specs):
            if sp.table is not None:                       # shares feature sp.table's table
                self.tables.append(self.tables[sp.table])
                continue
            users = [j for j, s in enumerate(specs) if j == k or s.table == k]
            ref = np.zeros(sp.V, dtype=bool)
            for j in users:
                p = self.per[j]
                ref[p["post"][p["ok"]]] = True
            tab = _nan((sp.V, sp.dim), dev)
            vals = torch.tensor(rng.randint(-8, 9, size=(sp.V, sp.dim)) * 0.25, dtype=torch.float32, device=dev)
            r = torch.tensor(ref, device=dev)
            tab[r] = vals[r]
            self.tables.append(tab)
        self.out = _nan((rows, self.ld), dev)

    # ---- descriptors ---------------------------------------------------------------------------------------
    def feature(self, k, out, src=None, table=None):
        K, L = _kern()
        sp = self.specs[k]
        ic, lc, wc, col = self.lay[k]
        ib = self.ids64 if sp.i64 else self.ids32
        return K.make_feature(
            self.tables[k] if table is None else table, ib[:self.B, ic:ic + sp.T], out, out_col=col,
            out_ld=self.ld, maxlen=sp.T,
            pool={"none": L.POOL_NONE, "sum": L.POOL_SUM, "mean": L.POOL_MEAN, "max": L.POOL_MAX}[sp.pool],
            mask_mode={"none": L.MASK_NONE, "zero": L.MASK_ZERO_ID, "length": L.MASK_LENGTH}[sp.mask],
            length=self.lenb[:self.B, lc] if lc is not None else None,
            weight=self.wb[:self.B, wc:wc + sp.T] if wc is not None else None,
            weight_mode={"none": L.WEIGHT_NONE, "raw": L.WEIGHT_RAW, "softmax": L.WEIGHT_SOFTMAX}[sp.weight],
            hash_mode={"none": L.HASH_NONE, "farm": L.HASH_FARM, "farm_mz": L.HASH_FARM_MASK_ZERO}[sp.hash],
            src_table=src, vocab=sp.V)

    def feats(self, out):
        return [self.feature(k, out) for k in range(len(self.specs))]

    def window_mask(self):
        m = torch.zeros((self.B + EXTRA, self.ld), dtype=torch.bool, device=self.dev)
        for sp, (_, _, _, col) in zip(self.specs, self.lay):
            m[:self.B, col:col + sp.width] = True
        return m

    # ---- float64 reference -------------------------------------------------------------------------------
    def parts(self, k):
        """(x [B,T,dim] fp32 rows (zero for out-of-range ids), weights [B,T] fp32, valid, ok, L fp32 [B])."""
        sp, p, dev = self.specs[k], self.per[k], self.dev
        tab = self.tables[k]
        post = torch.tensor(p["post"], device=dev)
        ok = torch.tensor(p["ok"], device=dev)
        valid = torch.tensor(p["valid"], device=dev)
        x = tab[torch.where(ok, post, torch.zeros_like(post))]
        x = torch.where(ok[:, :, None], x, torch.zeros_like(x))
        T = sp.T
        if sp.weight == "none":
            wt = torch.ones((self.B, T), device=dev)
        else:
            w = torch.tensor(p["w"], device=dev)
            if sp.weight == "raw":
                wt = torch.where(valid, w, torch.zeros_like(w))
            else:
                s = torch.where(valid, w, torch.full_like(w, NEG_PAD))
                win = s == s.max(1, keepdim=True).values          # exp(0) = 1, every other term underflows to 0
                n = win.sum(1, keepdim=True).float()
                wt = torch.where(win, 1.0 / n, torch.zeros_like(w))
        if sp.mask == "length":
            Lf = torch.tensor(p["ln"], device=dev).float()
        else:
            Lf = valid.sum(1).float()
        return x, wt, valid, ok, Lf

    def forward_values(self, k):
        """The fp32 values max pooling compares: x * w, and x * w - 1e9 at masked positions."""
        x, wt, valid, ok, Lf = self.parts(k)
        v = x * wt[:, :, None]
        return torch.where(valid[:, :, None], v, v - 1e9), v, wt, valid, ok, Lf

    def gather_ref(self, k):
        sp = self.specs[k]
        x, wt, valid, ok, Lf = self.parts(k)
        if sp.pool == "none":
            return x.reshape(self.B, -1).double()
        mv, v, wt, valid, ok, Lf = self.forward_values(k)
        if sp.pool == "max":
            assert bool((v.abs() < 32).all()), "masked max operands must stay below 32 to tie at -1e9"
            return mv.max(1).values.double()
        terms = (v * valid[:, :, None]).double()
        _on_grid(terms, "pooled terms")
        _fits(terms.abs().sum(1), "pooled sum")
        s = terms.sum(1)
        if sp.pool == "mean":
            s = (_f32(s) / (Lf + 1e-8)[:, None]).double()
        return s

    def max_shares(self, k, g):
        """(hit & ok, share = g / cnt * w in fp32) per [B, T, dim] position of max-pooled feature k."""
        mv, v, wt, valid, ok, Lf = self.forward_values(k)
        hit = mv == mv.max(1, keepdim=True).values
        cnt = hit.sum(1, keepdim=True).float()
        share = (g[:, None, :] / cnt) * wt[:, :, None]
        return hit & ok[:, :, None], share

    def grad(self, k, gen_scale=0.5):
        """An exact incoming gradient [B, width] for feature k (see the module docstring)."""
        sp, dev = self.specs[k], self.dev
        g = torch.tensor(self.rng.randint(-3, 4, size=(self.B, sp.width)) * gen_scale, dtype=torch.float32,
                         device=dev)
        if sp.pool == "mean":
            x, wt, valid, ok, Lf = self.parts(k)
            g = g * torch.where(Lf == 0, torch.ones_like(Lf), Lf.abs())[:, None]
        elif sp.pool == "max":
            mv, v, wt, valid, ok, Lf = self.forward_values(k)
            hit = mv == mv.max(1, keepdim=True).values
            g = g * hit.sum(1).float()
            if sp.weight == "softmax" and sp.T & (sp.T - 1):
                g[~valid.any(1)] = 0.0                                 # 1/T is not exact there
        return g

    def scatter_terms(self, k, g, scale=SCALE):
        """(row ids [N], terms [N, dim] float64) that a scatter of gradient g adds to feature k's table."""
        sp = self.specs[k]
        x, wt, valid, ok, Lf = self.parts(k)
        post = torch.tensor(self.per[k]["post"], device=self.dev)
        gs = g * scale
        if sp.pool == "none":
            sel = ok
            terms = gs.reshape(self.B, sp.T, sp.dim)
        elif sp.pool == "max":
            sel, share = self.max_shares(k, gs)
            terms = torch.where(sel, share, torch.zeros_like(share))
            sel = ok
        else:
            if sp.pool == "mean":
                gs = gs / (Lf + 1e-8)[:, None]
            terms = gs[:, None, :] * wt[:, :, None]
            sel = valid & ok
        return post[sel], terms[sel].double()

    def updated(self, tab, contribs, what):
        """tab + the sum of every (ids, terms), in float64, with the exact-range check."""
        t64 = tab.double().clone()
        bound = t64.abs().nan_to_num(0.0)
        for ids, terms in contribs:
            _on_grid(terms, what)
            t64.index_add_(0, ids, terms)
            bound.index_add_(0, ids, terms.abs())
        _fits(bound, what)
        return t64


def _check_gather(launch, what):
    K, L = _kern()
    K.embed_oob_count(reset=True)
    K.embed_gather_fwd(launch.feats(launch.out), launch.B)
    n = K.embed_oob_count(reset=True)
    for k, sp in enumerate(launch.specs):
        col = launch.lay[k][3]
        _same(launch.out[:launch.B, col:col + sp.width], launch.gather_ref(k), "%s: gather of feature %d (%s)"
              % (what, k, sp))
    outside = ~launch.window_mask()
    assert bool((_bits(launch.out)[outside] == NAN_BITS).all()), what + ": the gather wrote outside its windows"
    assert n == launch.n_oob, "%s: %d out-of-range ids counted, the reference visits %d" % (what, n, launch.n_oob)


def _check_scatter(launch, what, scale=SCALE):
    """Dense-target scatter (max pooling re-reads its forward rows from src_table): each table gets a copy of
    itself as the target, the forward tables are untouched."""
    K, L = _kern()
    gbuf = _nan((launch.B + EXTRA, launch.ld), launch.dev)
    gs = {}
    for k, sp in enumerate(launch.specs):
        col = launch.lay[k][3]
        gs[k] = launch.grad(k)
        gbuf[:launch.B, col:col + sp.width] = gs[k]
    gkeep = gbuf.clone()
    fwd_bits = [_bits(t).clone() for t in launch.tables]
    targets = {}
    for k, sp in enumerate(launch.specs):
        base = sp.table if sp.table is not None else k
        if base not in targets:
            targets[base] = launch.tables[base].clone()
    feats = [launch.feature(k, gbuf, src=launch.tables[k] if sp.pool == "max" else None,
                            table=targets[sp.table if sp.table is not None else k])
             for k, sp in enumerate(launch.specs)]
    K.embed_scatter_add(feats, launch.B, scale)
    assert torch.equal(_bits(gbuf), _bits(gkeep)), what + ": the scatter wrote into its gradient"
    for k, t in enumerate(launch.tables):
        assert torch.equal(_bits(t), fwd_bits[k]), what + ": the scatter wrote into a forward table"
    for base, tgt in targets.items():
        users = [k for k, sp in enumerate(launch.specs) if k == base or sp.table == base]
        want = launch.updated(launch.tables[base], [launch.scatter_terms(k, gs[k], scale) for k in users],
                              "%s: table %d" % (what, base))
        nanrow = torch.isnan(launch.tables[base]).all(1)
        assert torch.equal(_bits(tgt)[nanrow], _bits(launch.tables[base])[nanrow]), \
            "%s: the scatter changed a row no id references (table %d)" % (what, base)
        _same(tgt[~nanrow], want[~nanrow], "%s: scatter into table %d (%s)" % (what, base, launch.specs[base]))


def _run(specs, B, seed, what, cuda, ld_pad=5, scatter=True):
    lau = Launch(specs, B, seed, cuda, ld_pad=ld_pad)
    _check_gather(lau, what)
    if scatter:
        _check_scatter(lau, what)
    return lau


def _mix(dim, i64=False, odd=False):
    """All four pools at one dim: POOL_NONE, a length-masked sum, a zero-masked mean, a length-masked max."""
    return [Spec(dim, 3, "none", i64=i64, odd_col=odd), Spec(dim, 5, "sum", "length", "raw", i64=not i64, odd_col=odd),
            Spec(dim, 4, "mean", "zero", i64=i64, odd_col=odd), Spec(dim, 50, "max", "length", "softmax", odd_col=odd)]


# ================================================================================================ widths
@pytest.mark.parametrize("dim", [4, 8, 12, 16, 32, 64, 68, 128, 132, 256])
def test_vec4_widths(cuda, dim):
    _run(_mix(dim), 37, dim, "float4 dim %d" % dim, cuda, ld_pad=4)


@pytest.mark.parametrize("dim", [1, 2, 3, 5, 31, 33, 65, 130])
def test_scalar_widths(cuda, dim):
    _run(_mix(dim, i64=True), 37, 100 + dim, "scalar dim %d" % dim, cuda)


@pytest.mark.parametrize("how", ["out_col", "out_ld"])
def test_vec4_dims_forced_scalar(cuda, how):
    """dims % 4 == 0 whose out_col (or the row pitch) is not a multiple of 4 take the scalar path."""
    specs = _mix(8, odd=how == "out_col") + _mix(64)
    _run(specs, 41, 7, "forced scalar (%s)" % how, cuda, ld_pad=5 if how == "out_ld" else 4)


def test_widest_feature_sets_the_group(cuda):
    specs = [Spec(4, 3, "none"), Spec(256, 4, "max", "zero", "raw"), Spec(8, 5, "sum", "length"),
             Spec(1, 4, "mean", "length"), Spec(12, 1, "none", i64=True)]
    _run(specs, 53, 8, "narrow features at G 32 (float4)", cuda, ld_pad=4)
    specs = [Spec(1, 3, "none"), Spec(130, 4, "max", "zero", "raw"), Spec(2, 5, "sum", "length"),
             Spec(3, 4, "mean", "length")]
    _run(specs, 53, 9, "narrow features at G 32 (scalar)", cuda)


# ================================================================================================ modes
def test_pool_mask_weight_hash_matrix(cuda):
    """every pool x mask x weight, hashing and id widths cycled, in one launch (float4, dim 8)"""
    specs = []
    i = 0
    for pool in POOLS:
        for mask in MASKS:
            for weight in WEIGHTS:
                if pool == "none" and weight != "none":
                    continue
                specs.append(Spec(8, [3, 4, 5, 1][i % 4], pool, mask, weight, HASHES[i % 3], i64=i % 2 == 1,
                                  V=29 + i % 5))
                i += 1
    _run(specs, 67, 11, "pool x mask x weight (float4)", cuda, ld_pad=4)
    for sp in specs:
        sp.dim = 3
    _run(specs, 67, 12, "pool x mask x weight (scalar)", cuda)


@pytest.mark.parametrize("T", [1, 3, 4, 5, 50, 200])
def test_sequence_lengths(cuda, T):
    """every remainder of the gather's 4-position unroll, each pool and mask, hashed and plain"""
    specs = [Spec(4, T, "none", hash="farm"), Spec(8, T, "sum", "zero", "softmax"),
             Spec(4, T, "mean", "length", "raw", i64=True), Spec(8, T, "max", "zero", hash="farm_mz"),
             Spec(4, T, "max", "length", "softmax", i64=True), Spec(8, T, "max", "none", "raw")]
    _run(specs, 45, 20 + T, "T %d" % T, cuda, ld_pad=4)


# ================================================================================================ grid, chunks
@pytest.mark.parametrize("G,dim", [(1, 4), (8, 32), (32, 128)])
def test_grid_cap(cuda, G, dim):
    """tasks B * nfeat at cap - 1, cap, cap + 1 and past 2 * cap, cap = 1056 * 256 / G (two features)"""
    cap = NUM_SMS * 8 * 256 // G
    for n in (cap - 1, cap, cap + 1, 2 * cap + 3):
        B = (n + 1) // 2
        specs = [Spec(dim, 1, "none", V=1000), Spec(dim, 2, "max", "length", V=1000)]
        if 2 * B != n:
            specs = [Spec(dim, 3, "mean", "zero", V=1000)]
            B = n
        _run(specs, B, G + n, "G %d, %d tasks" % (G, B * len(specs)), cuda, ld_pad=4)


@pytest.mark.parametrize("nfeat", [63, 64, 65, 128])
def test_descriptor_chunks(cuda, nfeat):
    specs = []
    for i in range(nfeat):
        specs.append(Spec([4, 1, 8][i % 3], 1 + i % 4, POOLS[i % 4], MASKS[(i // 4) % 3], "raw" if i % 7 == 0 else
                          "none", i64=i % 2 == 0, V=13 + i % 7))
    _run(specs, 29, nfeat, "%d features" % nfeat, cuda)


# ================================================================================================ zero-row skip
@pytest.mark.parametrize("dim", [16, 132, 5, 8])
def test_pool_none_scatter_zero_rows(cuda, dim):
    """the POOL_NONE scatter skips a row whose gradient is all zero: zero rows next to nonzero ones in one warp,
    rows whose only nonzero sits in the last lane or the second pass, rows of -0.0"""
    K, L = _kern()
    B, T = 67, 5
    lau = Launch([Spec(dim, T, "none", V=11), Spec(dim, 1, "none", V=11, table=0)], B, 300 + dim, cuda, ld_pad=4)
    vec = dim % 4 == 0
    lanes = dim // 4 if vec else dim
    G = 1
    while G < lanes and G < 32:
        G *= 2
    rng = np.random.RandomState(dim)
    gbuf = _nan((B + EXTRA, lau.ld), cuda)
    gs = {}
    for k, sp in enumerate(lau.specs):
        g = torch.tensor(rng.randint(-3, 4, size=(B, sp.T, dim)) * 0.5, dtype=torch.float32)
        kind = rng.randint(0, 5, size=(B, sp.T))
        for b in range(B):
            for t in range(sp.T):
                if kind[b, t] == 0:
                    g[b, t] = 0.0
                elif kind[b, t] == 1:
                    g[b, t] = -0.0
                elif kind[b, t] == 2:                     # only the last element of the last lane's first pass
                    last = (min(G, lanes) * (4 if vec else 1)) - 1
                    g[b, t] = 0.0
                    g[b, t, min(last, dim - 1)] = 1.5
                elif kind[b, t] == 3:                     # only in the second pass (or the last element)
                    g[b, t] = 0.0
                    g[b, t, min(G * (4 if vec else 1), dim - 1)] = -2.0
        gs[k] = g.reshape(B, -1).to(cuda)
        col = lau.lay[k][3]
        gbuf[:B, col:col + sp.width] = gs[k]
    tgt = lau.tables[0].clone()
    K.embed_scatter_add([lau.feature(k, gbuf, table=tgt) for k in range(2)], B, SCALE)
    want = lau.updated(lau.tables[0], [lau.scatter_terms(k, gs[k]) for k in range(2)], "zero rows")
    nanrow = torch.isnan(lau.tables[0]).all(1)
    assert torch.equal(_bits(tgt)[nanrow], _bits(lau.tables[0])[nanrow])
    _same(tgt[~nanrow], want[~nanrow], "zero-row skip, dim %d" % dim)


# ================================================================================================ C4
def test_c4_shape(cuda):
    """DIN at C4: the [8192] query gather and the [8192, 50, 64] key gather from a 100,001-row table with Zipf
    ids, and the key gradients applied as 409,600 single-row lookups with half the rows' gradients zero"""
    K, L = _kern()
    B, T, E, V = 8192, 50, 64, 100001
    rng = np.random.RandomState(4)
    ln = rng.randint(1, T + 1, size=B)
    hist = _zipf(rng, V, (B, T), low=1)
    hist[np.arange(T)[None, :] >= ln[:, None]] = 0
    item = _zipf(rng, V, (B, 1), low=1)
    lau = Launch([Spec(E, 1, "none", V=V, oob=False), Spec(E, T, "none", V=V, oob=False, table=0)], B, 5, cuda,
                 ld_pad=4, ids={0: item, 1: hist})
    _check_gather(lau, "C4 gathers")
    # the flat key scatter: ids [B*T], gradient rows [B*T, E] of which half are zero
    ids = torch.tensor(hist.reshape(-1), dtype=torch.int32, device=cuda)
    n = B * T
    g = torch.tensor(rng.randint(-3, 4, size=(n, E)) * 0.5, dtype=torch.float32, device=cuda)
    g[torch.tensor(rng.rand(n) < 0.5, device=cuda)] = 0.0
    gbuf = _nan((n + EXTRA, E + 4), cuda)
    gbuf[:n, :E] = g
    tgt = lau.tables[0].clone()
    K.embed_scatter_add([K.make_feature(tgt, ids, gbuf[:n, :E], maxlen=1)], n, SCALE)
    want = lau.updated(lau.tables[0], [(ids.long(), (g * SCALE).double())], "C4 key scatter")
    nanrow = torch.isnan(lau.tables[0]).all(1)
    assert torch.equal(_bits(tgt)[nanrow], _bits(lau.tables[0])[nanrow])
    _same(tgt[~nanrow], want[~nanrow], "C4 flat key scatter")


# ================================================================================================ max in place
def _max_specs(vec4):
    """max-pooled bags of few-row tables (repeated arg-max ids within bags and across samples), one table shared
    with a sum-pooled bag; ``vec4``: dims that allow the float4 path"""
    if vec4:
        return [Spec(8, 6, "max", "zero", V=9), Spec(8, 5, "max", "length", "raw", V=9, table=0),
                Spec(8, 1, "sum", "none", V=9, table=0), Spec(64, 50, "max", "length", V=40),
                Spec(4, 3, "max", "none", "softmax", V=6, i64=True)]
    return [Spec(3, 6, "max", "zero", V=9), Spec(3, 5, "max", "length", "raw", V=9, table=0),
            Spec(3, 1, "sum", "none", V=9, table=0), Spec(3, 4, "max", "zero", "softmax", hash="farm_mz", V=7),
            Spec(5, 3, "max", "none", V=6, i64=True), Spec(33, 50, "max", "length", "raw", V=40)]


@pytest.mark.parametrize("vec4", [True, False])
@pytest.mark.parametrize("B", [7, 301])
def test_max_pool_fused_update_in_place(cuda, B, vec4):
    """Max pooling under the fused SGD update: the scatter refuses to re-find an arg-max at rows it writes (before
    any launch: the tables keep their bits); the shares are taken at the forward rows (every element of their
    window written, nothing outside, at a float4 pitch and at an odd one), and the POOL_NONE scatter applies them
    in place, in one launch with a sum-pooled bag of the same table.  The result is the reference update taken at
    the forward values."""
    K, L = _kern()
    lau = Launch(_max_specs(vec4), B, 40 + B, cuda, ld_pad=4)
    _check_gather(lau, "max bags")
    fwd = [t.clone() for t in lau.tables]
    maxk = [k for k, sp in enumerate(lau.specs) if sp.pool == "max"]
    gbuf = _nan((B + EXTRA, lau.ld), cuda)
    gs = {}
    for k, sp in enumerate(lau.specs):
        gs[k] = lau.grad(k)
        gbuf[:B, lau.lay[k][3]:lau.lay[k][3] + sp.width] = gs[k]
    for k in maxk:
        for src in (None, lau.tables[k]):
            with pytest.raises(ValueError, match="src_table"):
                K.embed_scatter_add([lau.feature(k, gbuf, src=src)], B, SCALE)
    assert all(torch.equal(_bits(a), _bits(b)) for a, b in zip(lau.tables, fwd)), "a refused scatter wrote"
    width = sum(lau.specs[k].T * lau.specs[k].dim for k in maxk)
    for pitch in (width + 4, width + 1):
        flat = _nan(((B + EXTRA) * pitch,), cuda)
        shares = flat[:B * pitch].view(B, pitch)[:, :width]
        K.embed_max_pool_shares([lau.feature(k, gbuf) for k in maxk], B, shares)
        col = 0
        for k in maxk:
            sp = lau.specs[k]
            hit, share = lau.max_shares(k, gs[k])
            want = torch.where(hit, share, torch.zeros_like(share)).reshape(B, -1).double()
            _same(shares[:, col:col + sp.T * sp.dim], want, "shares of feature %d (%s, pitch %d)" % (k, sp, pitch))
            col += sp.T * sp.dim
        inside = torch.zeros(flat.shape, dtype=torch.bool, device=cuda)
        inside[:B * pitch].view(B, pitch)[:, :width] = True
        assert bool((_bits(flat)[~inside] == NAN_BITS).all()), "shares written outside their window"
    assert all(torch.equal(_bits(a), _bits(b)) for a, b in zip(lau.tables, fwd)), "the shares wrote a table"
    feats, col = [], 0
    for k in maxk:
        sp = lau.specs[k]
        ic = lau.lay[k][0]
        ib = lau.ids64 if sp.i64 else lau.ids32
        feats.append(K.make_feature(lau.tables[k], ib[:B, ic:ic + sp.T], shares, out_col=col, out_ld=shares.stride(0),
                                    maxlen=sp.T, hash_mode=lau.feature(k, gbuf).hash_mode, vocab=sp.V))
        col += sp.T * sp.dim
    feats += [lau.feature(k, gbuf) for k, sp in enumerate(lau.specs) if sp.pool != "max"]
    K.embed_scatter_add(feats, B, SCALE)
    live, lau.tables = lau.tables, fwd              # the reference reads the forward values
    for base in sorted({sp.table if sp.table is not None else k for k, sp in enumerate(lau.specs)}):
        users = [k for k, sp in enumerate(lau.specs) if k == base or sp.table == base]
        want = lau.updated(fwd[base], [lau.scatter_terms(k, gs[k]) for k in users], "in-place table %d" % base)
        nanrow = torch.isnan(fwd[base]).all(1)
        assert torch.equal(_bits(live[base])[nanrow], _bits(fwd[base])[nanrow])
        _same(live[base][~nanrow], want[~nanrow], "fused max-pool update of table %d (B %d)" % (base, B))


def test_misaligned_src_table_takes_the_scalar_path(cuda):
    """a src_table view 4 bytes into its buffer (dim % 4 == 0, everything else aligned)"""
    K, L = _kern()
    lau = Launch([Spec(8, 5, "max", "length", "raw", V=9), Spec(16, 3, "max", "zero", V=9)], 33, 77, cuda, ld_pad=4)
    gbuf = _nan((lau.B + EXTRA, lau.ld), cuda)
    gs = {k: lau.grad(k) for k in range(2)}
    for k, sp in enumerate(lau.specs):
        gbuf[:lau.B, lau.lay[k][3]:lau.lay[k][3] + sp.width] = gs[k]
    for k, sp in enumerate(lau.specs):
        flat = _nan((sp.V * sp.dim + 8,), cuda)
        src = flat[1:1 + sp.V * sp.dim].view(sp.V, sp.dim)
        src.copy_(lau.tables[k])
        assert src.data_ptr() % 16 == 4
        tgt = lau.tables[k].clone()
        K.embed_scatter_add([lau.feature(k, gbuf, src=src, table=tgt)], lau.B, SCALE)
        want = lau.updated(lau.tables[k], [lau.scatter_terms(k, gs[k])], "misaligned src")
        nanrow = torch.isnan(lau.tables[k]).all(1)
        _same(tgt[~nanrow], want[~nanrow], "max scatter with a misaligned src_table (feature %d)" % k)


def test_deepfm_max_bag_sparse_equals_dense(cuda):
    """A DeepFM over one max-pooled VarLen feature (its embedding and its linear table), trained 2 SGD steps with
    embedding_update 'sparse' (the fused update writes the tables max pooling finds its arg-max in) and 'dense',
    from the same exact-valued weights with l2 = 0: the tables end bit-identical.  Every bag repeats an id, the 4
    samples share ids, and T = 2 keeps every tie count a power of two.  The model is linear in each trainable
    (one field: the FM term is zero; no hidden layer; mse with B = 4 and lr = 1/2), so both steps stay exact: the
    weights start on a 2^-1 grid, step 1 moves them on a 2^-6 grid, and step 2's updates are multiples of 2^-21
    on tables below 8 in magnitude."""
    from deepctr_b200.engine import SGD
    from deepctr_b200.feature_column import SparseFeat, VarLenSparseFeat
    from deepctr_b200.models import DeepFM
    from deepctr_b200 import ops
    rng = np.random.RandomState(3)
    cols = [VarLenSparseFeat(SparseFeat("hist", 3, 4), maxlen=2, combiner="max")]
    x = {"hist": np.array([[1, 1], [2, 2], [1, 2], [2, 0]], dtype=np.int32)}
    y = np.array([1.0, -0.5, 0.5, 0.0], dtype=np.float32)
    init = None
    tables = {}
    ops.set_gemm_precision("fp32")
    try:
        for mode in ("sparse", "dense"):
            model = DeepFM(cols, cols, dnn_hidden_units=(), l2_reg_linear=0, l2_reg_embedding=0, task="regression")
            if init is None:
                init = [(rng.randint(-2, 3, size=w.shape) * 0.5).astype(np.float32) for w in model.weights]
            for w, v in zip(model.weights, init):
                w.set_value(v)
            model.compile(SGD(0.5), "mse", embedding_update=mode)
            for _ in range(2):
                model.train_on_batch(x, y)
            tables[mode] = {w.name: w.value() for w in model.weights if "emb" in w.name}
    finally:
        ops.set_gemm_precision("bf16x3")
    assert len(tables["sparse"]) == 2 and tables["sparse"].keys() == tables["dense"].keys()
    for name, want in tables["dense"].items():
        got = tables["sparse"][name]
        diff = np.abs(got.astype(np.float64) - want).max()
        assert np.array_equal(got.view(np.int32), want.view(np.int32)), \
            "table %s: the fused update differs from the dense one by up to %g" % (name, diff)


def test_onn_max_bag_sparse_update_equals_dense_gradient(cuda):
    """ONN's field-aware tables of a max-pooled VarLen field under the fused update: one SGD step of 'sparse' moves
    every table by -lr x the 'dense' gradient taken at the pre-step weights.  Every bag repeats an id and 5 rows
    serve 512 samples.  The products make the gradients inexact, and red.add sums a row's terms in any order: the
    tolerance is test_onn_gpu's (1e-4 relative), far below the half of a tied gradient the update must not drop."""
    from deepctr_b200 import engine as E_, models as M
    from deepctr_b200.engine import SGD
    from deepctr_b200.feature_column import SparseFeat, VarLenSparseFeat
    lr, n = 0.05, 512
    res, init = {}, None
    for mode in ("dense", "sparse"):
        rng = np.random.RandomState(9)
        cols = [SparseFeat("C%d" % i, 5, 4) for i in range(3)] + \
            [VarLenSparseFeat(SparseFeat("bag", 5, 4), maxlen=4, combiner="max")]
        bag = rng.randint(1, 5, size=(n, 4)).astype(np.int32)
        bag[:, 1] = bag[:, 0]
        bag[rng.rand(n, 4) < 0.25] = 0
        x = {"C%d" % i: rng.randint(0, 5, size=n).astype(np.int32) for i in range(3)}
        x["bag"] = bag
        y = (rng.rand(n) < 0.3).astype(np.float32)
        E_.clear_session()
        model = M.ONN(cols, cols, dnn_hidden_units=(8,), l2_reg_embedding=0, l2_reg_linear=0, use_bn=False)
        if init is None:
            init = [(rng.normal(0, 0.3, size=w.shape)).astype(np.float32) for w in model.weights]
        model.set_weights(init)
        model.compile(SGD(lr), "binary_crossentropy", embedding_update=mode, step_graph="off")
        model.train_on_batch(x, y)
        assert any(f[2] == 3 for f in model.planner.ffm.fields), "the bag is not a max-pooled field-aware field"
        res[mode] = {t.embeddings.name: t.embeddings.value() for _, t in model.planner.ffm.tables}
    w0 = dict(zip([w.name for w in model.weights], init))
    bags = [k for k in res["dense"] if "bag" in k]
    assert bags
    for k in res["dense"]:
        d_dense = res["dense"][k] - w0[k]
        d_sparse = res["sparse"][k] - w0[k]
        np.testing.assert_allclose(d_sparse, d_dense, rtol=1e-4, atol=1e-6 * max(1.0, float(np.abs(d_dense).max())),
                                   err_msg=k)
        assert np.abs(d_dense).max() > 0, k


# ================================================================================================ masks
def _bytes_buf(n, dev):
    return torch.full((n + 4099,), 0x5a, dtype=torch.uint8, device=dev)


@pytest.mark.parametrize("B,T", [(5, 7), (THREAD_CAP // 50 + 1, 50), (3, THREAD_CAP // 3 + 2)])
def test_mask_from_len(cuda, B, T):
    """out[b, t] = t < len[b] for lengths < 0, 0, T, > T; n across the thread cap; bytes past n unchanged"""
    K, L = _kern()
    rng = np.random.RandomState(B)
    ln = rng.randint(-2, T + 3, size=B).astype(np.int32)
    ln[:min(B, 5)] = [-(1 << 31), 0, T, T + 1, -1][:min(B, 5)]
    lens = torch.tensor(ln, device=cuda)
    buf = _bytes_buf(B * T, cuda)
    L.check(L.lib().b2ctr_mask_from_len(K.ptr(lens), B, T, K.ptr(buf), K.stream()), "mask_from_len")
    want = (torch.arange(T, device=cuda)[None, :] < lens[:, None].long()).to(torch.uint8).reshape(-1)
    assert torch.equal(buf[:B * T], want), "mask_from_len (B %d, T %d)" % (B, T)
    assert bool((buf[B * T:] == 0x5a).all()), "mask_from_len wrote past n"


@pytest.mark.parametrize("n", [1, 7, THREAD_CAP - 1, THREAD_CAP, THREAD_CAP + 1, 2 * THREAD_CAP + 5])
@pytest.mark.parametrize("dtype", [torch.int32, torch.int64])
def test_mask_nonzero_and(cuda, n, dtype):
    """first: ids != 0; then AND into the mask (bytes 1, 2, 255, 0 going in); int64 ids nonzero only in their high
    32 bits count as nonzero; bytes past n unchanged"""
    K, L = _kern()
    rng = np.random.RandomState(n)
    ids = rng.randint(-3, 4, size=n).astype(np.int64)
    if dtype == torch.int64:
        hi = rng.rand(n) < 0.2
        high = np.array([1 << 32, -(1 << 32), 1 << 62, 5 << 32], dtype=np.int64)
        ids[hi] = high[rng.randint(0, 4, size=int(hi.sum()))]
    else:
        ids[rng.rand(n) < 0.05] = INT32_MIN
    idt = torch.tensor(ids, device=cuda).to(dtype)
    nz = torch.tensor(ids != 0, device=cuda)
    buf = _bytes_buf(n, cuda)
    lib = L.lib()
    L.check(lib.b2ctr_mask_nonzero_and(K.ptr(idt), K.idx_dtype(idt), n, K.ptr(buf), 1, K.stream()), "mask")
    assert torch.equal(buf[:n], nz.to(torch.uint8)), "mask_nonzero_and (first)"
    assert bool((buf[n:] == 0x5a).all())
    prior = torch.tensor(np.array([0, 1, 2, 255], dtype=np.uint8)[rng.randint(0, 4, size=n)], device=cuda)
    buf[:n] = prior
    L.check(lib.b2ctr_mask_nonzero_and(K.ptr(idt), K.idx_dtype(idt), n, K.ptr(buf), 0, K.stream()), "mask")
    assert torch.equal(buf[:n], prior & nz.to(torch.uint8)), "mask_nonzero_and (AND)"
    assert bool((buf[n:] == 0x5a).all()), "mask_nonzero_and wrote past n"


# ================================================================================================ pack_rows
@pytest.mark.parametrize("widths,batch", [([1], 9), ([3, 1], 17), ([1] * 62 + [131], 5), ([2, 7] * 32, 33),
                                          ([1] * 63 + [5], 3), ([13], THREAD_CAP // 13 + 1),
                                          ([1, 300], THREAD_CAP // 301 * 2 + 7)])
def test_pack_rows(cuda, widths, batch):
    """dst[b, col_i + c] = block_i[b, c] at a pitch ld_dst > total; the gaps and rows past the batch keep their NaN"""
    K, L = _kern()
    total = sum(widths)
    rng = np.random.RandomState(len(widths) + batch)
    blocks = [torch.tensor(rng.randint(-99, 100, size=(batch, w)) * 0.5, dtype=torch.float32) for w in widths]
    src = torch.cat([b.reshape(-1) for b in blocks] + [_nan((7,), "cpu")]).to(cuda)
    ld = total + 3
    dst = _nan((batch + EXTRA, ld), cuda)
    arr = (C.c_int32 * len(widths))(*widths)
    L.check(L.lib().b2ctr_pack_rows(K.ptr(src), arr, len(widths), batch, K.ptr(dst), ld, K.stream()), "pack_rows")
    want = torch.cat(blocks, 1).to(cuda)
    assert torch.equal(dst[:batch, :total], want), "pack_rows (%d blocks, batch %d)" % (len(widths), batch)
    assert bool((_bits(dst[:batch, total:]) == NAN_BITS).all()) and bool((_bits(dst[batch:]) == NAN_BITS).all()), \
        "pack_rows wrote outside [batch, total]"


# ================================================================================================ hashing
def _decimal_ids(rng):
    """ids of every decimal length 1..20 (with the sign), both signs, plus the int64 / int32 extremes"""
    out = [0]
    for d in range(1, 20):
        lo, hi = 10 ** (d - 1), 10 ** d - 1
        for v in (lo, hi, int(rng.randint(0, 1 << 62) % (hi - lo + 1)) + lo):
            out += [v, -v]
    out += [(1 << 63) - 1, -(1 << 63), -(1 << 63) + 1, 10 ** 18, -10 ** 18]
    return [v for v in out if -(1 << 63) <= v < (1 << 63)]


def test_hash64_every_decimal_length(cuda):
    K, L = _kern()
    rng = np.random.RandomState(17)
    ids = np.array(_decimal_ids(rng), dtype=np.int64)
    lens = {len(str(int(v))) for v in ids}
    assert lens == set(range(1, 21)), sorted(lens)
    i32 = np.array([v for v in ids if -(1 << 31) <= v < (1 << 31)] + [INT32_MIN, (1 << 31) - 1, -1], dtype=np.int32)
    for nb, mz in [(1, False), (2, True), (1 << 20, False), (1 << 20, True), ((1 << 63) - 25, False),
                   ((1 << 63) - 25, True)]:
        want = np.array([farmhash.hash_bucket(int(v), nb, mz) for v in ids], dtype=np.int64)
        got = K.hash64(torch.tensor(ids, device=cuda), nb, mz).cpu().numpy()
        assert np.array_equal(got, want), "hash64 int64, num_buckets %d, mask_zero %s" % (nb, mz)
        want32 = np.array([farmhash.hash_bucket(int(v), nb, mz) for v in i32], dtype=np.int64)
        got32 = K.hash64(torch.tensor(i32, device=cuda), nb, mz).cpu().numpy()
        assert np.array_equal(got32, want32), "hash64 int32 (sign extended), num_buckets %d, mask_zero %s" % (nb, mz)


@pytest.mark.parametrize("i64", [False, True])
def test_in_kernel_hash_every_decimal_length(cuda, i64):
    """the gather hashes in the kernel: the ids of every decimal length as one POOL_NONE sequence and one summed bag
    per sample, into 61 buckets, 2 buckets with mask_zero and 1 bucket"""
    rng = np.random.RandomState(18)
    ids = np.array(_decimal_ids(rng), dtype=np.int64)
    if not i64:
        ids = np.array([v for v in ids if -(1 << 31) <= v < (1 << 31)] + [INT32_MIN], dtype=np.int64)
    seq = np.stack([np.roll(ids, s) for s in range(3)])
    for V, h in ((61, "farm"), (2, "farm_mz"), (1, "farm")):
        lau = Launch([Spec(4, len(ids), "none", hash=h, V=V, i64=i64),
                      Spec(3, len(ids), "sum", "zero" if h == "farm_mz" else "none", hash=h, V=V, i64=i64)],
                     3, 19, cuda, ld_pad=4, ids={0: seq, 1: seq})
        _check_gather(lau, "in-kernel hash, %d buckets (%s, %s)" % (V, h, "int64" if i64 else "int32"))
