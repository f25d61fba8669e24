"""Thin, autograd-free wrappers: torch CUDA tensors in, C-ABI call, torch CUDA tensors out.

torch only provides device memory (``torch.empty``) and the current stream handle here; every
byte of arithmetic happens inside libb2ctr.so.  These functions are what the GPU parity tests
call ("through the C-ABI") and what the engine (``engine.py``) builds its tape ops from.
"""
import contextlib
import ctypes as C
import functools

import torch

from . import _lib as L

_workspace = {}
_retired = []


def _require_cuda(*tensors):
    for t in tensors:
        if t is not None and not t.is_cuda:
            raise L.B2ctrError("b2ctr kernels need CUDA tensors: there is no CPU fallback")


def stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


def workspace(nbytes, device):
    """Grow-only scratch buffer per device (caller-provided workspace of the C-ABI)."""
    if nbytes <= 0:
        return None
    key = (device.index if device.index is not None else torch.cuda.current_device())
    buf = _workspace.get(key)
    if buf is None or buf.numel() < nbytes:
        if buf is not None:
            _retired.append(buf)      # captured step graphs may still reference the old scratch: keep it
        size = max(nbytes, 1 << 20, 2 * buf.numel() if buf is not None else 0)
        if torch.cuda.is_current_stream_capturing():
            raise RuntimeError("workspace growth during CUDA-graph capture (run the step eagerly first)")
        buf = torch.empty(size, dtype=torch.uint8, device=device)
        _workspace[key] = buf
    return buf


def idx_dtype(t):
    if t.dtype == torch.int32:
        return L.IDX_I32
    if t.dtype == torch.int64:
        return L.IDX_I64
    raise ValueError("ids must be int32 or int64, got %s" % t.dtype)


# ---- optional per-kernel timing (bench.py): CUDA events around each launch on the launching stream --
PROFILE = None
PROFILE_TAG = None       # set by `profile_tag(...)`: the launch is recorded as "<tag>:<wrapper name>"


@contextlib.contextmanager
def profiled():
    """Record the launches of a block into a fresh PROFILE dict, which is yielded; PROFILE is None again after."""
    global PROFILE
    PROFILE = {}
    try:
        yield PROFILE
    finally:
        PROFILE = None


class profile_tag(object):
    """Attribute the launches of a region (CIN layers, the DIN attention unit ...) to a named group."""

    def __init__(self, tag):
        self.tag = tag

    def __enter__(self):
        global PROFILE_TAG
        self.prev, PROFILE_TAG = PROFILE_TAG, (self.tag if PROFILE_TAG is None else PROFILE_TAG)

    def __exit__(self, *a):
        global PROFILE_TAG
        PROFILE_TAG = self.prev


def _timed(fn):
    """Decorate a wrapper that enqueues device work: while PROFILE is a dict, each call records one CUDA-event
    pair around it under the wrapper's name."""
    name = fn.__name__

    @functools.wraps(fn)
    def wrap(*a, **k):
        prof = PROFILE
        if prof is None:
            return fn(*a, **k)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        r = fn(*a, **k)
        e1.record()
        prof.setdefault(name if PROFILE_TAG is None else "%s:%s" % (PROFILE_TAG, name), []).append((e0, e1))
        return r

    return wrap


def profile_summary():
    """{kernel wrapper name: (launch groups, total ms)} for everything recorded into PROFILE."""
    torch.cuda.synchronize()
    out = {}
    for name, evs in (PROFILE or {}).items():
        out[name] = (len(evs), float(sum(a.elapsed_time(b) for a, b in evs)))
    return out


# ---- embedding ------------------------------------------------------------------------------
def make_feature(table, idx, out, out_col=0, out_ld=None, maxlen=1, pool=L.POOL_NONE,
                 mask_mode=L.MASK_NONE, length=None, weight=None, weight_mode=L.WEIGHT_NONE,
                 hash_mode=L.HASH_NONE, idx_stride=None, src_table=None, vocab=None):
    """Fill one b2ctr_feature_t.  ``idx`` is [B] / [B,1] / [B,T] (or a strided column view).  ``vocab``:
    the FULL vocabulary when ``table`` is only a shard of it (ids are validated against it)."""
    _require_cuda(table, idx, out)
    f = L.Feature()
    f.table = table.data_ptr()
    f.idx = idx.data_ptr()
    f.len = length.data_ptr() if length is not None else None
    f.weight = weight.data_ptr() if weight is not None else None
    # side inputs may be column windows of a packed staging buffer: pass their sample strides
    f.len_stride = length.stride(0) if (length is not None and length.dim() >= 1 and length.shape[0] > 1) else 0
    f.weight_ld = weight.stride(0) if (weight is not None and weight.dim() >= 2 and weight.shape[0] > 1) else 0
    f.out = out.data_ptr()
    f.vocab = table.shape[0] if vocab is None else int(vocab)
    f.dim = table.shape[1] if table.dim() > 1 else 1
    f.idx_stride = idx_stride if idx_stride is not None else (idx.stride(0) if idx.dim() >= 1 else 1)
    f.out_ld = out_ld if out_ld is not None else out.stride(0)
    f.out_col = out_col
    f.maxlen = maxlen
    f.idx_dtype = idx_dtype(idx)
    f.pool = pool
    f.mask_mode = mask_mode
    f.hash_mode = hash_mode
    f.weight_mode = weight_mode
    f.src_table = src_table.data_ptr() if src_table is not None else None
    return f


def _feat_array(feats):
    arr = (L.Feature * len(feats))(*feats)
    return arr


@_timed
def embed_gather_fwd(feats, batch):
    arr = _feat_array(feats)
    L.check(L.lib().b2ctr_embed_gather_fwd(arr, len(feats), batch, stream()), "embed_gather_fwd")


def embed_oob_count(reset=True):
    """Number of embedding ids outside [0, vocabulary_size) the gather kernels of this device have seen
    (they read a zero row and are skipped by the updates).  Synchronises the current stream."""
    n = C.c_int64(0)
    L.check(L.lib().b2ctr_embed_oob_count(C.byref(n), 1 if reset else 0, stream()), "embed_oob_count")
    return int(n.value)


@_timed
def embed_scatter_add(feats, batch, scale):
    arr = _feat_array(feats)
    L.check(L.lib().b2ctr_embed_scatter_add(arr, len(feats), batch, scale, stream()),
            "embed_scatter_add")


@_timed
def embed_max_pool_shares(feats, batch, shares):
    """Max pooling's backward per position: feature f's [T*dim] block of ``shares`` (a [batch, >= sum T*dim] view)
    starts at the sum of the preceding features' T*dim; see b2ctr_embed_max_pool_shares."""
    _require_cuda(shares)
    arr = _feat_array(feats)
    L.check(L.lib().b2ctr_embed_max_pool_shares(arr, len(feats), batch, ptr(shares), shares.stride(0), stream()),
            "embed_max_pool_shares")


class UniformPlan(object):
    """Host-side descriptor for the Criteo-shaped fast path; keeps ctypes arrays alive."""

    def __init__(self, feats, lin_tables, dense, x, linear, fm, fm_mask):
        self.feat_arr = _feat_array(feats)
        self.g = L.UniformGather()
        self.g.feats = self.feat_arr
        if lin_tables is not None:
            self.lin_arr = (C.c_void_p * len(feats))(*[t.data_ptr() for t in lin_tables])
            self.g.lin_tables = self.lin_arr
        self.g.dense = dense.data_ptr() if dense is not None else None
        self.g.x = x.data_ptr()
        self.g.linear = linear.data_ptr() if linear is not None else None
        self.g.fm = fm.data_ptr() if fm is not None else None
        self.g.ldx = x.stride(0)
        self.g.dense_ld = dense.stride(0) if dense is not None else 0
        self.g.nfeat = len(feats)
        self.g.ndense = dense.shape[1] if dense is not None else 0
        self.g.fm_mask[0] = fm_mask & 0xFFFFFFFFFFFFFFFF
        self.g.fm_mask[1] = 0
        # with the FM fused: the gather also stores S [B, dim], which the scatter then reads instead of re-summing x
        self.fm_sum = (torch.empty((x.shape[0], feats[0].dim), dtype=torch.float32, device=x.device)
                       if fm is not None else None)
        self.x_rows, self.x_device = x.shape[0], x.device
        self.x_planes, self.x_planes_cols = None, 0

    def set_planes(self, cols):
        """Have the gather also write the bf16 operand planes (split_planes layout) of x[:, :cols]; returns them."""
        nbytes = L.lib().b2ctr_planes_bytes(self.x_rows, cols)
        self.x_planes = torch.empty((nbytes,), dtype=torch.uint8, device=self.x_device)
        self.x_planes_cols = cols
        return self.x_planes

    def set_peers(self, world, peer_tables, peer_lin_tables):
        """Row-sharded tables addressed through peer mappings (parallel.PeerTables.table device arrays)."""
        self.peer_refs = (peer_tables, peer_lin_tables)
        self.g.world = world
        self.g.peer_tables = peer_tables.data_ptr()
        self.g.peer_lin_tables = peer_lin_tables.data_ptr() if peer_lin_tables is not None else None


@_timed
def embed_gather_uniform_fwd(plan, batch):
    L.check(L.lib().b2ctr_embed_gather_uniform_fwd_ex(C.byref(plan.g), ptr(plan.fm_sum), ptr(plan.x_planes),
                                                      plan.x_planes_cols, batch, stream()),
            "embed_gather_uniform_fwd")


@_timed
def embed_scatter_uniform_bwd(plan, dx, dfm, dlinear, scale, lin_scale, batch, fm_sum=None):
    """``fm_sum``: the S [B, dim] a gather of the same x stored (UniformPlan.fm_sum), or None: the scatter sums x."""
    L.check(L.lib().b2ctr_embed_scatter_uniform_bwd_ex(C.byref(plan.g), ptr(dx), ptr(dfm), ptr(fm_sum),
                                                       ptr(dlinear), scale, lin_scale, batch, stream()),
            "embed_scatter_uniform_bwd")


@_timed
def embed_update_sorted(plan, dx, dfm, dlinear, optimizer, lr, lin_lr, eps, acc_tables, lin_acc_tables, batch):
    """Deterministic fused update (sort by (table, id) + ordered segmented reduce, one write per row):
    optimizer 0 = SGD, 1 = Keras Adagrad (lazy / sparse apply) with per-element accumulators."""
    nf = plan.g.nfeat
    dim = plan.feat_arr[0].dim
    nbytes = L.lib().b2ctr_embed_update_sorted_workspace_bytes(nf, dim, batch)
    dev = dx.device if dx is not None else (dfm.device if dfm is not None else dlinear.device)
    ws = workspace(nbytes, dev)
    acc = (C.c_void_p * nf)(*[t.data_ptr() for t in acc_tables]) if acc_tables is not None else None
    lacc = (C.c_void_p * nf)(*[t.data_ptr() for t in lin_acc_tables]) if lin_acc_tables is not None else None
    L.check(L.lib().b2ctr_embed_update_sorted(C.byref(plan.g), ptr(dx), ptr(dfm), ptr(dlinear), optimizer, lr, lin_lr,
                                              eps, acc, lacc, batch, ptr(ws), nbytes, stream()),
            "embed_update_sorted")


@_timed
def hash64(ids, num_buckets, mask_zero):
    _require_cuda(ids)
    ids = ids.contiguous()
    out = torch.empty(ids.shape, dtype=torch.int64, device=ids.device)
    L.check(L.lib().b2ctr_hash64(ptr(ids), idx_dtype(ids), ids.numel(), num_buckets,
                                 1 if mask_zero else 0, ptr(out), stream()), "hash64")
    return out


@_timed
def init_normal(dst, mean, std, seed):
    _require_cuda(dst)
    L.check(L.lib().b2ctr_init_normal(ptr(dst), dst.numel(), mean, std, seed, stream()), "init_normal")
    return dst


# ---- GEMM -----------------------------------------------------------------------------------
@_timed
def gemm(a, b, c=None, bias=None, trans_a=False, trans_b=False, act=L.ACT_NONE, accumulate=False,
         precision=L.GEMM_FP32, split_k=1, alpha=1.0, m=None, n=None, k=None, variant=0, a_planes=None,
         b_planes=None):
    """C[M,N] = act(alpha * op(A) @ op(B) + bias) on 2-D row-major (possibly ld-padded) tensors.

    In BF16X3 mode an fp32 operand may be None when its planes are given (m, n, k then required); the call raises
    ValueError, before any launch, if it would have to split that operand itself."""
    _require_cuda(a, b, c, bias, a_planes, b_planes)
    if (a is None and a_planes is None) or (b is None and b_planes is None):
        raise ValueError("gemm: an fp32 operand may be None only when its planes are given")
    if (a is None or b is None) and None in (m, n, k):
        raise ValueError("gemm: m, n and k are required when an fp32 operand is None")
    if m is None:
        m = a.shape[1] if trans_a else a.shape[0]
    if k is None:
        k = a.shape[0] if trans_a else a.shape[1]
    if n is None:
        n = b.shape[0] if trans_b else b.shape[1]
    dev = next(t.device for t in (a, b, a_planes, b_planes) if t is not None)
    if c is None:
        c = torch.empty((m, n), dtype=torch.float32, device=dev)
    g = L.Gemm()
    g.a = a.data_ptr() if a is not None else None
    g.b = b.data_ptr() if b is not None else None
    g.c = c.data_ptr()
    g.bias = bias.data_ptr() if bias is not None else None
    g.m, g.n, g.k = m, n, k
    # (a missing operand gets the smallest leading dimension the C-ABI accepts; it is never read)
    g.lda = a.stride(0) if a is not None else (m if trans_a else k)
    g.ldb = b.stride(0) if b is not None else (k if trans_b else n)
    g.ldc = c.stride(0)
    g.trans_a, g.trans_b = int(trans_a), int(trans_b)
    g.act, g.accumulate, g.precision, g.split_k, g.alpha = act, int(accumulate), precision, split_k, alpha
    g.variant = variant
    g.a_planes = a_planes.data_ptr() if a_planes is not None else None
    g.b_planes = b_planes.data_ptr() if b_planes is not None else None
    nbytes = L.lib().b2ctr_gemm_workspace_bytes(C.byref(g))
    ws = workspace(nbytes, dev)
    L.check(L.lib().b2ctr_gemm(C.byref(g), ptr(ws), nbytes if ws is not None else 0, stream()), "gemm")
    return c


@_timed
def split_planes(x2d):
    """bf16 hi/lo planes of a 2-D fp32 tensor (row stride may exceed the width) for BF16X3 GEMMs."""
    _require_cuda(x2d)
    rows, cols = x2d.shape
    nbytes = L.lib().b2ctr_planes_bytes(rows, cols)
    buf = torch.empty((nbytes,), dtype=torch.uint8, device=x2d.device)
    L.check(L.lib().b2ctr_split_planes(ptr(x2d), x2d.stride(0), rows, cols, ptr(buf), stream()), "split_planes")
    return buf


# ---- elementwise ----------------------------------------------------------------------------
def planes_fusable(m, n):
    """bias_act_bwd can write the operand planes of dz itself (no padding inside the planes, vector layout)."""
    return m % 256 == 0 and (n == 64 or n % 128 == 0) and n % 4 == 0 and n // 4 <= 256 and 256 % (n // 4) == 0


@_timed
def bias_act_bwd(dy, y, act, want_dz=True, want_dbias=True, m=None, n=None, want_planes=False):
    """dz = dy * act'(y), dbias = colsum(dz); with want_planes also the bf16 operand planes of dz
    (returned as third value)."""
    _require_cuda(dy, y)
    if m is None:
        m, n = dy.shape[0], dy.shape[1]
    ld = dy.stride(0)
    # one row pitch for dy, y and dz: a strided dy (a window of a wider buffer) gets a dz window with the same pitch
    if y is not None and y.dim() == 2 and y.stride(0) != ld:
        raise ValueError("bias_act_bwd: dy and y must have the same row pitch (%d != %d)" % (ld, y.stride(0)))
    dz = torch.empty((m, ld), dtype=torch.float32, device=dy.device)[:, :n] if want_dz else None
    dbias = torch.empty((n,), dtype=torch.float32, device=dy.device) if want_dbias else None
    nbytes = L.lib().b2ctr_bias_act_bwd_workspace_bytes(m, n) if want_dbias else 0
    ws = workspace(nbytes, dy.device)
    if want_planes:
        planes = torch.empty((L.lib().b2ctr_planes_bytes(m, n),), dtype=torch.uint8, device=dy.device)
        L.check(L.lib().b2ctr_bias_act_bwd_planes(ptr(dy), ptr(y), ptr(dz), ptr(dbias), ptr(planes), m, n, ld, act,
                                                  ptr(ws), nbytes, stream()), "bias_act_bwd_planes")
        return dz, dbias, planes
    L.check(L.lib().b2ctr_bias_act_bwd(ptr(dy), ptr(y), ptr(dz), ptr(dbias), m, n, ld, act, ptr(ws),
                                       nbytes, stream()), "bias_act_bwd")
    return dz, dbias


# ---- fused relu tower (hidden layers 1..L-1 of a DNN) -----------------------------------------
def _widths(widths):
    return (C.c_int32 * len(widths))(*widths), len(widths)


def _ptrs(ts):
    return (C.c_void_p * len(ts))(*[t.data_ptr() if t is not None else None for t in ts])


def _planes(rows, cols, device):
    return torch.empty((L.lib().b2ctr_planes_bytes(rows, cols),), dtype=torch.uint8, device=device)


@_timed
def mlp_relu_fwd(y0, ws, bs):
    """y_i = relu(y_{i-1} W_i + b_i) for the layers after y0 [B, n0] (b2ctr_mlp_relu_fwd).  Returns the planes of
    y_0 .. y_{L-2} and y_{L-1}."""
    _require_cuda(y0, *ws, *bs)
    widths = [y0.shape[1]] + [w.shape[1] for w in ws]
    m = y0.shape[0]
    planes = [_planes(m, n, y0.device) for n in widths[:-1]]
    y = torch.empty((m, widths[-1]), dtype=torch.float32, device=y0.device)
    L.check(L.lib().b2ctr_mlp_relu_fwd(ptr(y0.contiguous()), _ptrs(ws), _ptrs(bs), _ptrs(planes), ptr(y),
                                       *_widths(widths), m, stream()), "mlp_relu_fwd")
    return planes, y


@_timed
def mlp_relu_bwd(dy, y, y0, planes, ws):
    """The backward of mlp_relu_fwd from dy = d y_{L-1} (b2ctr_mlp_relu_bwd): the planes of dz_0 .. dz_{L-1} and
    the bias gradients db_0 .. db_{L-1}."""
    _require_cuda(dy, y, y0, *ws)
    widths = [y0.shape[1]] + [w.shape[1] for w in ws]
    m = y0.shape[0]
    dzp = [_planes(m, n, y0.device) for n in widths]
    db = [torch.empty((n,), dtype=torch.float32, device=y0.device) for n in widths]
    wid = _widths(widths)
    nbytes = L.lib().b2ctr_mlp_relu_bwd_workspace_bytes(*wid)
    wsp = workspace(nbytes, y0.device)
    L.check(L.lib().b2ctr_mlp_relu_bwd(ptr(dy.contiguous()), ptr(y), ptr(y0), _ptrs(planes), _ptrs(ws), _ptrs(dzp),
                                       _ptrs(db), *wid, m, ptr(wsp), nbytes, stream()), "mlp_relu_bwd")
    return dzp, db


@_timed
def act_fwd(x, act, out=None):
    _require_cuda(x)
    out = torch.empty_like(x) if out is None else out
    L.check(L.lib().b2ctr_act_fwd(ptr(x), ptr(out), x.numel(), act, stream()), "act_fwd")
    return out


@_timed
def add_n(ins, scales=None, out=None):
    _require_cuda(*ins)
    out = torch.empty_like(ins[0]) if out is None else out
    arr = (C.c_void_p * len(ins))(*[t.data_ptr() for t in ins])
    sc = (C.c_float * len(ins))(*(scales if scales is not None else [1.0] * len(ins)))
    L.check(L.lib().b2ctr_add_n(arr, sc, len(ins), ptr(out), out.numel(), stream()), "add_n")
    return out


@_timed
def axpy(x, y, alpha=1.0):
    _require_cuda(x, y)
    L.check(L.lib().b2ctr_axpy(ptr(x), ptr(y), alpha, x.numel(), stream()), "axpy")
    return y


@_timed
def fill(dst, value):
    _require_cuda(dst)
    L.check(L.lib().b2ctr_fill(ptr(dst), value, dst.numel(), stream()), "fill")
    return dst


@_timed
def mask_nonzero_and(ids, inout=None):
    """uint8 mask [B,T] of ids != 0, AND-ed into ``inout`` when given."""
    _require_cuda(ids, inout)
    first = inout is None
    if first:
        inout = torch.empty(ids.shape, dtype=torch.uint8, device=ids.device)
    L.check(L.lib().b2ctr_mask_nonzero_and(ptr(ids), idx_dtype(ids), ids.numel(), ptr(inout), int(first),
                                           stream()), "mask_nonzero_and")
    return inout


@_timed
def mask_from_len(lengths, maxlen):
    _require_cuda(lengths)
    lengths = lengths.reshape(-1)
    out = torch.empty((lengths.shape[0], maxlen), dtype=torch.uint8, device=lengths.device)
    L.check(L.lib().b2ctr_mask_from_len(ptr(lengths), lengths.shape[0], maxlen, ptr(out), stream()),
            "mask_from_len")
    return out


@_timed
def copy2d(src, ld_src, dst, ld_dst, rows, cols, accumulate=False, src_off=0, dst_off=0):
    _require_cuda(src, dst)
    sp = C.c_void_p(src.data_ptr() + 4 * src_off)
    dp = C.c_void_p(dst.data_ptr() + 4 * dst_off)
    L.check(L.lib().b2ctr_copy2d(sp, ld_src, dp, ld_dst, rows, cols, int(accumulate), stream()), "copy2d")
    return dst


@_timed
def pack_rows(src_flat, widths, batch, out=None):
    """[sum_i B*w_i] flat blocks -> row-major [B, sum w_i]."""
    _require_cuda(src_flat)
    total = int(sum(widths))
    if out is None:
        out = torch.empty((batch, total), dtype=torch.float32, device=src_flat.device)
    arr = (C.c_int32 * len(widths))(*[int(w) for w in widths])
    L.check(L.lib().b2ctr_pack_rows(ptr(src_flat), arr, len(widths), batch, ptr(out), total, stream()), "pack_rows")
    return out


@_timed
def rowsum(x, rows, cols, ld=None):
    _require_cuda(x)
    out = torch.empty((rows,), dtype=torch.float32, device=x.device)
    L.check(L.lib().b2ctr_rowsum(ptr(x), ld if ld is not None else x.stride(0), ptr(out), rows, cols,
                                 stream()), "rowsum")
    return out


@_timed
def fm_fwd(x, nfield, dim, ldx=None):
    _require_cuda(x)
    batch = x.shape[0]
    out = torch.empty((batch,), dtype=torch.float32, device=x.device)
    L.check(L.lib().b2ctr_fm_fwd(ptr(x), ldx if ldx is not None else x.stride(0), nfield, dim, ptr(out),
                                 batch, stream()), "fm_fwd")
    return out


@_timed
def fm_bwd(x, nfield, dim, dout, dx=None, accumulate=False, ldx=None):
    _require_cuda(x, dout)
    batch = x.shape[0]
    ldx = ldx if ldx is not None else x.stride(0)
    if dx is None:
        dx = torch.empty_like(x)
        accumulate = False
    L.check(L.lib().b2ctr_fm_bwd(ptr(x), ldx, nfield, dim, ptr(dout), ptr(dx), dx.stride(0),
                                 int(accumulate), batch, stream()), "fm_bwd")
    return dx


@_timed
def fm_weighted_fwd(x, ldx, m, nfield, dim, batch):
    """FM of m ⊙ x: x a [B, nfield*dim] window (row pitch ldx), m [B, nfield] (row pitch m.stride(0)) -> [B]."""
    _require_cuda(x, m)
    out = torch.empty((batch,), dtype=torch.float32, device=x.device)
    L.check(L.lib().b2ctr_fm_weighted_fwd(ptr(x), ldx, ptr(m), m.stride(0), nfield, dim, ptr(out), batch, stream()),
            "fm_weighted_fwd")
    return out


@_timed
def fm_weighted_bwd(x, ldx, m, nfield, dim, dout, batch, dx=None, accumulate=False, want_dx=True, want_dm=True):
    """(dx [B, nfield*dim] or the given window, dm [B, nfield] | None).  ``dx`` given: written with its own row pitch,
    added to when ``accumulate``."""
    _require_cuda(x, m, dout, dx)
    if dx is None and want_dx:
        dx = torch.empty((batch, nfield * dim), dtype=torch.float32, device=x.device)
        accumulate = False
    dm = torch.empty((batch, nfield), dtype=torch.float32, device=x.device) if want_dm else None
    L.check(L.lib().b2ctr_fm_weighted_bwd(ptr(x), ldx, ptr(m), m.stride(0), nfield, dim, ptr(dout), ptr(dx),
                                          dx.stride(0) if dx is not None else nfield * dim, int(accumulate), ptr(dm),
                                          nfield, batch, stream()), "fm_weighted_bwd")
    return dx, dm


@_timed
def field_scale_fwd(x, ldx, m, nfield, dim, batch, out=None):
    """y[b, f*dim + e] = x[b, f*dim + e] * m[b, f] -> [B, nfield*dim] (or into ``out``, a 2-D window)."""
    _require_cuda(x, m, out)
    if out is None:
        out = torch.empty((batch, nfield * dim), dtype=torch.float32, device=x.device)
    L.check(L.lib().b2ctr_field_scale_fwd(ptr(x), ldx, ptr(m), m.stride(0), nfield, dim, ptr(out), out.stride(0),
                                          batch, stream()), "field_scale_fwd")
    return out


@_timed
def field_scale_bwd(dy, x, ldx, m, nfield, dim, batch, dx=None, accumulate=False, want_dx=True, want_dm=True):
    """(dx = dy * m [B, nfield*dim] or the given window, dm = sum_e dy x [B, nfield] | None)."""
    _require_cuda(dy, x, m, dx)
    if dx is None and want_dx:
        dx = torch.empty((batch, nfield * dim), dtype=torch.float32, device=x.device)
        accumulate = False
    dm = torch.empty((batch, nfield), dtype=torch.float32, device=x.device) if want_dm else None
    L.check(L.lib().b2ctr_field_scale_bwd(ptr(dy), dy.stride(0), ptr(x), ldx, ptr(m), m.stride(0), nfield, dim,
                                          ptr(dx), dx.stride(0) if dx is not None else nfield * dim, int(accumulate),
                                          ptr(dm), nfield, batch, stream()), "field_scale_bwd")
    return dx, dm


@_timed
def softmax_rows_fwd(x, scale=1.0):
    """scale * softmax along the rows of a 2-D window x (row pitch x.stride(0)) -> a new [rows, cols] tensor."""
    _require_cuda(x)
    rows, cols = x.shape
    y = torch.empty((rows, cols), dtype=torch.float32, device=x.device)
    L.check(L.lib().b2ctr_softmax_rows_fwd(ptr(x), x.stride(0), ptr(y), cols, rows, cols, scale, stream()),
            "softmax_rows_fwd")
    return y


@_timed
def softmax_rows_bwd(y, dy, scale=1.0):
    """dx = y * (dy - sum_j y_j dy_j / scale) for 2-D windows y, dy -> a new [rows, cols] tensor."""
    _require_cuda(y, dy)
    rows, cols = y.shape
    dx = torch.empty((rows, cols), dtype=torch.float32, device=y.device)
    L.check(L.lib().b2ctr_softmax_rows_bwd(ptr(y), y.stride(0), ptr(dy), dy.stride(0), ptr(dx), cols, rows, cols,
                                           scale, stream()), "softmax_rows_bwd")
    return dx


# ---- head / loss / optimizers ---------------------------------------------------------------
@_timed
def predict_loss(logit, bias=None, labels=None, task=L.TASK_BINARY, want_grad=False):
    """Returns (pred[B], dlogit[B] | None, dbias[1] | None, loss_sum[1] | None)."""
    _require_cuda(logit, bias, labels)
    batch = logit.numel()
    pred = torch.empty((batch,), dtype=torch.float32, device=logit.device)
    dlogit = torch.empty((batch,), dtype=torch.float32, device=logit.device) if want_grad else None
    acc = None
    if labels is not None:
        acc = torch.empty((2,), dtype=torch.float32, device=logit.device)
        fill(acc, 0.0)
    loss_sum = acc[0:1] if acc is not None else None
    dbias = acc[1:2] if (acc is not None and want_grad and bias is not None) else None
    L.check(L.lib().b2ctr_predict_loss(ptr(logit), ptr(bias), ptr(labels), ptr(pred), ptr(dlogit),
                                       ptr(dbias), ptr(loss_sum), batch, task, stream()), "predict_loss")
    return pred, dlogit, dbias, loss_sum


@_timed
def sgd_step(w, g, lr, l2=0.0):
    _require_cuda(w, g)
    L.check(L.lib().b2ctr_sgd_step(ptr(w), ptr(g), lr, l2, w.numel(), stream()), "sgd_step")


@_timed
def sgd_step_multi(ws, gs, lr, l2s):
    """w -= lr * (g + 2 l2 w) for a list of tensors in one launch."""
    n = len(ws)
    if n == 0:
        return
    _require_cuda(*ws)
    _require_cuda(*gs)
    wp, gp = (C.c_void_p * n)(*[ptr(t) for t in ws]), (C.c_void_p * n)(*[ptr(t) for t in gs])
    nn = (C.c_int64 * n)(*[t.numel() for t in ws])
    ll = (C.c_float * n)(*[float(v) for v in l2s])
    L.check(L.lib().b2ctr_sgd_step_multi(wp, gp, nn, ll, n, lr, stream()), "sgd_step_multi")


@_timed
def adam_step(w, g, m, v, lr, step, beta1=0.9, beta2=0.999, eps=1e-7, l2=0.0):
    _require_cuda(w, g, m, v)
    L.check(L.lib().b2ctr_adam_step(ptr(w), ptr(g), ptr(m), ptr(v), lr, beta1, beta2, eps, l2, step,
                                    w.numel(), stream()), "adam_step")


@_timed
def adam_step_dev(w, g, m, v, lr, step_dev, beta1=0.9, beta2=0.999, eps=1e-7, l2=0.0):
    """Adam with the step count read from the device tensor `step_dev` (int64 [1]): graph-replayable."""
    _require_cuda(w, g, m, v, step_dev)
    L.check(L.lib().b2ctr_adam_step_dev(ptr(w), ptr(g), ptr(m), ptr(v), lr, beta1, beta2, eps, l2, ptr(step_dev),
                                        w.numel(), stream()), "adam_step_dev")


@_timed
def counter_add(counter, delta=1):
    _require_cuda(counter)
    L.check(L.lib().b2ctr_counter_add(ptr(counter), delta, stream()), "counter_add")


@_timed
def adagrad_step(w, g, acc, lr, eps=1e-7, l2=0.0):
    _require_cuda(w, g, acc)
    L.check(L.lib().b2ctr_adagrad_step(ptr(w), ptr(g), ptr(acc), lr, eps, l2, w.numel(), stream()),
            "adagrad_step")


# ---- field-aware pairwise products (ONN) ---------------------------------------------------------------
def ffm_field(idx=None, vocab=1, hash_mode=L.HASH_NONE, pooled=None, grad=None):
    """One b2ctr_ffm_field_t: a single-valued field's ids [B] (or a strided column), or a pooled operand [B, ld]
    holding its F-1 per-partner rows; ``grad`` [B, ld] receives the backward's per-partner gradient rows."""
    _require_cuda(idx, pooled, grad)
    f = L.FfmField()
    if idx is not None:
        f.idx, f.idx_stride, f.idx_dtype = idx.data_ptr(), idx.stride(0), idx_dtype(idx)
        f.vocab, f.hash_mode = int(vocab), hash_mode
    if pooled is not None:
        f.pooled, f.pooled_ld = pooled.data_ptr(), pooled.stride(0)
    if grad is not None:
        f.grad, f.grad_ld = grad.data_ptr(), grad.stride(0)
    return f


@_timed
def ffm_product_fwd(fields, tables, dim, reduce_sum, out, out_col, batch):
    """prod_p = e_{i,(j)} * e_{j,(i)} for every pair into ``out`` [B, ld] from column ``out_col``; ``tables`` the
    device int64 array [F*F] of table pointers."""
    arr = (L.FfmField * len(fields))(*fields)
    _lib_call("ffm_product_fwd", arr, len(fields), ptr(tables), dim, int(reduce_sum), ptr(out), out.stride(0),
              out_col, batch, stream())


@_timed
def ffm_product_bwd(fields, tables, dim, reduce_sum, g, g_col, batch):
    """Per-lookup gradient rows into each field's ``grad`` buffer, read at the tables' current values."""
    arr = (L.FfmField * len(fields))(*fields)
    _lib_call("ffm_product_bwd", arr, len(fields), ptr(tables), dim, int(reduce_sum), ptr(g), g.stride(0), g_col,
              batch, stream())


# ---- interaction / sequence operators ---------------------------------------------------------------
def _lib_call(name, *args):
    L.check(getattr(L.lib(), "b2ctr_" + name)(*args), name)


@_timed
def ewise(op, a, b, c=None, out=None, accumulate=False):
    _require_cuda(a, b, c, out)
    out = torch.empty_like(a) if out is None else out
    _lib_call("ewise", op, ptr(a), ptr(b), ptr(c), ptr(out), a.numel(), int(accumulate), stream())
    return out


@_timed
def cross_vector_fwd(x0, ld0, xl, ldl, w, bias, batch, dim):
    out = torch.empty((batch, dim), dtype=torch.float32, device=x0.device)
    s = torch.empty((batch,), dtype=torch.float32, device=x0.device)
    _lib_call("cross_vector_fwd", ptr(x0), ld0, ptr(xl), ldl, ptr(w), ptr(bias), ptr(out), ptr(s), batch, dim,
              stream())
    return out, s


@_timed
def cross_vector_bwd(x0, ld0, w, dout, s, batch, dim):
    dx0 = torch.empty((batch, dim), dtype=torch.float32, device=x0.device)
    dxl = torch.empty((batch, dim), dtype=torch.float32, device=x0.device)
    ds = torch.empty((batch,), dtype=torch.float32, device=x0.device)
    _lib_call("cross_vector_bwd", ptr(x0), ld0, ptr(w), ptr(dout), ptr(s), ptr(dx0), ptr(dxl), ptr(ds), batch,
              dim, stream())
    return dx0, dxl, ds


def _off(t, elems):
    return C.c_void_p(t.data_ptr() + 4 * elems)


@_timed
def cin_outer_fwd(x0, v0, xk, vk, z, b0, nb, m, h, d):
    """v0 / vk = (sb, si, sd) element strides; b0 = first sample of the chunk."""
    _lib_call("cin_outer_fwd", _off(x0, b0 * v0[0]), v0[0], v0[1], v0[2], _off(xk, b0 * vk[0]), vk[0], vk[1],
              vk[2], ptr(z), nb, m, h, d, stream())


@_timed
def cin_outer_bwd(dz, x0, v0, xk, vk, dx0, g0, acc0, dxk, gk, acck, b0, nb, m, h, d, hp=0):
    _lib_call("cin_outer_bwd", ptr(dz), _off(x0, b0 * v0[0]), v0[0], v0[1], v0[2], _off(xk, b0 * vk[0]), vk[0],
              vk[1], vk[2], _off(dx0, b0 * g0[0]) if dx0 is not None else C.c_void_p(0), g0[0], g0[1], g0[2],
              int(acc0), _off(dxk, b0 * gk[0]) if dxk is not None else C.c_void_p(0), gk[0], gk[1], gk[2],
              int(acck), nb, m, h, d, hp, stream())


@_timed
def cin_t0(x0, v0, nb, m, d, ld0):
    """T0[(b,d), i] = X0(b,i,d), zero-padded to ld0 columns: the per-row factors of the generated outer product."""
    t0 = torch.empty((nb * d, ld0), dtype=torch.float32, device=x0.device)
    _lib_call("cin_t0", ptr(x0), v0[0], v0[1], v0[2], ptr(t0), ld0, nb, m, d, stream())
    return t0


@_timed
def cin_filter_planes(w2d, m, h, hp):
    """bf16 hi/lo planes of the filter in the padded layout W'[i*hp + j, n] (w2d: [m*h, n])."""
    n = w2d.shape[1]
    planes = torch.empty((L.lib().b2ctr_cin_filter_planes_bytes(m, hp, n),), dtype=torch.uint8, device=w2d.device)
    _lib_call("cin_filter_planes", ptr(w2d), m, h, hp, n, ptr(planes), stream())
    return planes


@_timed
def cin_gemm(mode, t0, xk, ldk, rows, m, h, hp, n, planes, bias=None, act=L.ACT_NONE, split_k=1, out=None):
    """mode 0: Y[rows, n] = act(Z W' + bias) with planes = cin_filter_planes; mode 1: dW'[m*hp, n] = Z^T dY with
    planes = split_planes(dY).  Z[r, i*hp+j] = t0[r,i] * xk[r,j] is generated inside the GEMM producer."""
    g = L.CinGemm()
    g.t0, g.ld0, g.xk, g.ldk, g.rows = t0.data_ptr(), t0.stride(0), xk.data_ptr(), ldk, rows
    g.m, g.h, g.hp, g.n = m, h, hp, n
    g.w_planes = planes.data_ptr() if mode == 0 else None
    g.dy_planes = planes.data_ptr() if mode == 1 else None
    if out is None:
        out = torch.empty((rows if mode == 0 else m * hp, n), dtype=torch.float32, device=t0.device)
    g.c, g.ldc = out.data_ptr(), out.stride(0)
    g.bias = bias.data_ptr() if bias is not None else None
    g.act, g.mode, g.split_k = act, mode, split_k
    nbytes = L.lib().b2ctr_cin_gemm_workspace_bytes(C.byref(g))
    ws = workspace(nbytes, t0.device)
    L.check(L.lib().b2ctr_cin_gemm(C.byref(g), ptr(ws), nbytes, stream()), "cin_gemm")
    return out


@_timed
def att_gemm(mode, q2d, ldq, keys2d, key_batch_stride, batch, T, E, n, planes, bias=None, act=L.ACT_NONE, split_k=1):
    """First LocalActivationUnit layer with its [q, k, q-k, q*k] input generated inside the GEMM producer.
    mode 0: [B*T, n] = act(A W + bias) (planes of W [4E, n]); mode 1: [4E, n] = A^T dY (planes of dY [B*T, n])."""
    g = L.AttGemm()
    g.query, g.ldq, g.keys, g.key_batch_stride = q2d.data_ptr(), ldq, keys2d.data_ptr(), key_batch_stride
    g.batch, g.maxlen, g.dim, g.n = batch, T, E, n
    g.planes = planes.data_ptr()
    out = torch.empty((batch * T if mode == 0 else 4 * E, n), dtype=torch.float32, device=q2d.device)
    g.c, g.ldc = out.data_ptr(), n
    g.bias = bias.data_ptr() if bias is not None else None
    g.act, g.mode, g.split_k = act, mode, split_k
    nbytes = L.lib().b2ctr_att_gemm_workspace_bytes(C.byref(g))
    ws = workspace(nbytes, q2d.device)
    L.check(L.lib().b2ctr_att_gemm(C.byref(g), ptr(ws), nbytes, stream()), "att_gemm")
    return out


@_timed
def cin_fold(t0, xk, ldk, rows, m, h, hp, n, w_planes, dy_planes, dt0, dxk, ldx):
    """dZ = dY W'^T folded onto the factors inside the GEMM epilogue: dt0 [rows, ld0] and dxk [rows, ldx] are
    accumulated (zero them first; layer 0: dxk is dt0)."""
    g = L.CinGemm()
    g.t0, g.ld0, g.xk, g.ldk, g.rows = t0.data_ptr(), t0.stride(0), xk.data_ptr(), ldk, rows
    g.m, g.h, g.hp, g.n = m, h, hp, n
    g.w_planes, g.dy_planes = w_planes.data_ptr(), dy_planes.data_ptr()
    L.check(L.lib().b2ctr_cin_fold(C.byref(g), ptr(dt0), ptr(dxk), ldx, stream()), "cin_fold")


@_timed
def cin_t0_bwd(dt0, ld0, dx, gx, accumulate, nb, m, d):
    _lib_call("cin_t0_bwd", ptr(dt0), ld0, ptr(dx), gx[0], gx[1], gx[2], int(accumulate), nb, m, d, stream())


@_timed
def cin_unpad_rows(src, m, h, hp):
    n = src.shape[1]
    dst = torch.empty((m * h, n), dtype=torch.float32, device=src.device)
    _lib_call("cin_unpad_rows", ptr(src), ptr(dst), m, h, hp, n, stream())
    return dst


@_timed
def cin_sum_d(y, ldy, col0, ncols, d, out, ldo, out_col, b0, nb):
    _lib_call("cin_sum_d", ptr(y), ldy, col0, ncols, d, _off(out, b0 * ldo), ldo, out_col, nb, stream())


@_timed
def cin_expand_grad(dout, ldo, out_col, col0, ncols, dh, ldh, hcols, dy, nfilt, d, b0, nb):
    _lib_call("cin_expand_grad", _off(dout, b0 * ldo), ldo, out_col, col0, ncols, ptr(dh), ldh, hcols, ptr(dy),
              nfilt, d, nb, stream())


@_timed
def interacting_fwd(q, k, v, res, batch, F, H, D, scaling):
    out = torch.empty_like(q)
    _lib_call("interacting_fwd", ptr(q), ptr(k), ptr(v), ptr(res), ptr(out), batch, F, H, D, int(scaling),
              stream())
    return out


@_timed
def interacting_bwd(q, k, v, out, dout, want_res, batch, F, H, D, scaling):
    dq, dk, dv = torch.empty_like(q), torch.empty_like(q), torch.empty_like(q)
    dres = torch.empty_like(q) if want_res else None
    _lib_call("interacting_bwd", ptr(q), ptr(k), ptr(v), ptr(out), ptr(dout), ptr(dq), ptr(dk), ptr(dv),
              ptr(dres), batch, F, H, D, int(scaling), stream())
    return dq, dk, dv, dres


@_timed
def bi_interaction_fwd(x, ldx, nfield, dim, batch):
    """[B, nfield*dim] window (pitch ldx) -> [B, dim]:  0.5 * ((sum_f x)^2 - sum_f x^2)."""
    _require_cuda(x)
    out = torch.empty((batch, dim), dtype=torch.float32, device=x.device)
    _lib_call("bi_interaction_fwd", ptr(x), ldx, nfield, dim, ptr(out), dim, batch, stream())
    return out


@_timed
def bi_interaction_bwd(x, ldx, nfield, dim, g, batch):
    _require_cuda(x, g)
    dx = torch.empty((batch, nfield * dim), dtype=torch.float32, device=x.device)
    _lib_call("bi_interaction_bwd", ptr(x), ldx, nfield, dim, ptr(g), g.stride(0), ptr(dx), nfield * dim, batch,
              stream())
    return dx


@_timed
def afm_fwd(x, ldx, nfield, dim, W, bias, h, batch):
    """AFM attention pooling -> (att [B, dim], softmax state [B, 2])."""
    _require_cuda(x, W, bias, h)
    factor = W.shape[1]
    att = torch.empty((batch, dim), dtype=torch.float32, device=x.device)
    state = torch.empty((batch, 2), dtype=torch.float32, device=x.device)
    _lib_call("afm_fwd", ptr(x), ldx, nfield, dim, factor, ptr(W), ptr(bias), ptr(h), ptr(att), dim, ptr(state),
              batch, stream())
    return att, state


@_timed
def afm_bwd(g, x, ldx, nfield, dim, W, bias, h, state, att, batch):
    """-> (dx [B, nfield*dim], dW [dim, factor], dbias [factor], dh [factor])."""
    _require_cuda(g, x, W, bias, h, state, att)
    factor = W.shape[1]
    dev = x.device
    dx = torch.empty((batch, nfield * dim), dtype=torch.float32, device=dev)
    dW = torch.empty((dim, factor), dtype=torch.float32, device=dev)
    db = torch.empty((factor,), dtype=torch.float32, device=dev)
    dh = torch.empty((factor,), dtype=torch.float32, device=dev)
    nbytes = L.lib().b2ctr_afm_bwd_workspace_bytes(dim, factor, batch)
    ws = workspace(nbytes, dev)
    _lib_call("afm_bwd", ptr(g), g.stride(0), ptr(x), ldx, nfield, dim, factor, ptr(W), ptr(bias), ptr(h),
              ptr(state), ptr(att), att.stride(0), ptr(dx), nfield * dim, ptr(dW), ptr(db), ptr(dh), batch, ptr(ws),
              nbytes, stream())
    return dx, dW, db, dh


@_timed
def senet_fwd(x, ldx, nfield, dim, W1, W2, batch):
    """SENETLayer on a [B, nfield*dim] window (pitch ldx) -> (V [B, nfield*dim], saved (A1, A2) [B, R + nfield])."""
    _require_cuda(x, W1, W2)
    reduce = W1.shape[1]
    v = torch.empty((batch, nfield * dim), dtype=torch.float32, device=x.device)
    saved = torch.empty((batch, reduce + nfield), dtype=torch.float32, device=x.device)
    _lib_call("senet_fwd", ptr(x), ldx, nfield, dim, reduce, ptr(W1), ptr(W2), ptr(v), nfield * dim, ptr(saved),
              batch, stream())
    return v, saved


@_timed
def senet_bwd(g, x, ldx, nfield, dim, W1, W2, saved, batch):
    """-> (dx [B, nfield*dim], dW1 [nfield, R], dW2 [R, nfield])."""
    _require_cuda(g, x, W1, W2, saved)
    reduce = W1.shape[1]
    dev = x.device
    dx = torch.empty((batch, nfield * dim), dtype=torch.float32, device=dev)
    dW1 = torch.empty((nfield, reduce), dtype=torch.float32, device=dev)
    dW2 = torch.empty((reduce, nfield), dtype=torch.float32, device=dev)
    nbytes = L.lib().b2ctr_senet_bwd_workspace_bytes(nfield, reduce, batch)
    ws = workspace(nbytes, dev)
    _lib_call("senet_bwd", ptr(g), g.stride(0), ptr(x), ldx, nfield, dim, reduce, ptr(W1), ptr(W2), ptr(saved),
              ptr(dx), nfield * dim, ptr(dW1), ptr(dW2), batch, ptr(ws), nbytes, stream())
    return dx, dW1, dW2


BILINEAR_TYPES = {"all": 0, "each": 1, "interaction": 2}


@_timed
def bilinear_fwd(x, ldx, nfield, dim, btype, W, batch, out=None, col0=0, pitch=None):
    """BilinearInteraction on a [B, nfield*dim] window (pitch ldx) with the stacked weights W [nW, dim, dim].
    Pair p goes to columns [col0 + p*pitch, +dim) of ``out`` [B, ld] (default: a new [B, P*dim])."""
    _require_cuda(x, W)
    P = nfield * (nfield - 1) // 2
    if out is None:
        out = torch.empty((batch, P * dim), dtype=torch.float32, device=x.device)
    pitch = dim if pitch is None else pitch
    _lib_call("bilinear_fwd", ptr(x), ldx, nfield, dim, BILINEAR_TYPES[btype], ptr(W), ptr(out), out.stride(0), col0,
              pitch, batch, stream())
    return out


@_timed
def bilinear_bwd(g, ldg, gcol0, gpitch, x, ldx, nfield, dim, btype, W, batch, want_dx=True, want_dw=True):
    """g: the data pointer of the gradient buffer addressed like the forward's output -> (dx [B, nfield*dim], dW)."""
    _require_cuda(g, x, W)
    dev = x.device
    dx = torch.empty((batch, nfield * dim), dtype=torch.float32, device=dev) if want_dx else None
    dW = torch.empty(tuple(W.shape), dtype=torch.float32, device=dev) if want_dw else None
    nbytes = L.lib().b2ctr_bilinear_bwd_workspace_bytes(nfield, dim, batch) if want_dw else 0
    ws = workspace(nbytes, dev) if want_dw else None
    _lib_call("bilinear_bwd", ptr(g), ldg, gcol0, gpitch, ptr(x), ldx, nfield, dim, BILINEAR_TYPES[btype], ptr(W),
              ptr(dx), nfield * dim, ptr(dW), batch, ptr(ws), nbytes, stream())
    return dx, dW


@_timed
def fwfm_fwd(x, ldx, nfield, dim, r, batch):
    """FwFMLayer on a [B, nfield*dim] window (pitch ldx) with the strengths r [nfield, nfield] -> [B, 1]."""
    _require_cuda(x, r)
    out = torch.empty((batch, 1), dtype=torch.float32, device=x.device)
    _lib_call("fwfm_fwd", ptr(x), ldx, nfield, dim, ptr(r), ptr(out), 1, batch, stream())
    return out


@_timed
def fwfm_bwd(g, ldg, x, ldx, nfield, dim, r, batch, want_dx=True, want_dr=True):
    """-> (dx [B, nfield*dim] or None, dR [nfield, nfield] or None)."""
    _require_cuda(g, x, r)
    dev = x.device
    dx = torch.empty((batch, nfield * dim), dtype=torch.float32, device=dev) if want_dx else None
    dR = torch.empty((nfield, nfield), dtype=torch.float32, device=dev) if want_dr else None
    nbytes = L.lib().b2ctr_fwfm_bwd_workspace_bytes(nfield, batch) if want_dr else 0
    ws = workspace(nbytes, dev) if want_dr else None
    _lib_call("fwfm_bwd", ptr(g), ldg, ptr(x), ldx, nfield, dim, ptr(r), ptr(dx), nfield * dim, ptr(dR), batch,
              ptr(ws), nbytes, stream())
    return dx, dR


@_timed
def fefm_sym(W):
    """S_p = W_p + W_p^T for the stacked weights W [P, dim, dim]."""
    _require_cuda(W)
    S = torch.empty_like(W)
    _lib_call("fefm_sym", ptr(W), W.shape[0], W.shape[1], ptr(S), stream())
    return S


@_timed
def fefm_fwd(x, ldx, nfield, dim, S, batch, out=None, col0=0):
    """FEFMLayer on a [B, nfield*dim] window (pitch ldx) with S from fefm_sym: pair p's score goes to column
    col0 + p of ``out`` [B, ld] (default: a new [B, P])."""
    _require_cuda(x, S, out)
    if out is None:
        out = torch.empty((batch, nfield * (nfield - 1) // 2), dtype=torch.float32, device=x.device)
    _lib_call("fefm_fwd", ptr(x), ldx, nfield, dim, ptr(S), ptr(out), out.stride(0), col0, batch, stream())
    return out


@_timed
def fefm_bwd(g, ldg, gcol0, x, ldx, nfield, dim, S, batch, want_dx=True, want_dw=True):
    """g: the data pointer of the gradient buffer addressed like the forward's output -> (dx [B, nfield*dim] or
    None, dW [P, dim, dim] or None)."""
    _require_cuda(g, x, S)
    dev = x.device
    dx = torch.empty((batch, nfield * dim), dtype=torch.float32, device=dev) if want_dx else None
    dW = torch.empty(tuple(S.shape), dtype=torch.float32, device=dev) if want_dw else None
    nbytes = L.lib().b2ctr_fefm_bwd_workspace_bytes(nfield, dim, batch) if want_dw else 0
    ws = workspace(nbytes, dev) if want_dw else None
    _lib_call("fefm_bwd", ptr(g), ldg, gcol0, ptr(x), ldx, nfield, dim, ptr(S), ptr(dx), nfield * dim, ptr(dW), batch,
              ptr(ws), nbytes, stream())
    return dx, dW


PNN_MODES = {"inner": 0, "elementwise": 1, "vec": 2, "num": 3}   # b2ctr.h B2CTR_PNN_*


@_timed
def pnn_inner_fwd(x, ldx, nfield, dim, mode, Kw, batch, out=None, col0=0):
    """InnerProductLayer / OutterProductLayer('vec' | 'num') on a [B, nfield*dim] window (pitch ldx); ``mode`` a
    PNN_MODES key, ``Kw`` the kernel (None for 'inner' / 'elementwise').  The pair scores (P*dim products for
    'elementwise') go to columns col0.. of ``out`` [B, ld] (default: a new [B, P] or [B, P*dim])."""
    _require_cuda(x, Kw, out)
    m = PNN_MODES[mode]
    if out is None:
        P = nfield * (nfield - 1) // 2
        out = torch.empty((batch, P * dim if mode == "elementwise" else P), dtype=torch.float32, device=x.device)
    _lib_call("pnn_inner_fwd", ptr(x), ldx, nfield, dim, m, ptr(Kw), ptr(out), out.stride(0), col0, batch, stream())
    return out


@_timed
def pnn_inner_bwd(g, ldg, gcol0, x, ldx, nfield, dim, mode, Kw, batch, want_dx=True, want_dk=True):
    """g: the data pointer of the gradient buffer addressed like the forward's output -> (dx [B, nfield*dim] or
    None, dK shaped like Kw or None)."""
    _require_cuda(g, x, Kw)
    dev = x.device
    m = PNN_MODES[mode]
    want_dk = want_dk and mode in ("vec", "num")
    dx = torch.empty((batch, nfield * dim), dtype=torch.float32, device=dev) if want_dx else None
    dK = torch.empty(tuple(Kw.shape), dtype=torch.float32, device=dev) if want_dk else None
    nbytes = L.lib().b2ctr_pnn_inner_bwd_workspace_bytes(nfield, dim, m, batch) if want_dk else 0
    ws = workspace(nbytes, dev) if want_dk else None
    _lib_call("pnn_inner_bwd", ptr(g), ldg, gcol0, ptr(x), ldx, nfield, dim, m, ptr(Kw), ptr(dx), nfield * dim,
              ptr(dK), batch, ptr(ws), nbytes, stream())
    return dx, dK


@_timed
def pnn_outer_fwd(x, ldx, nfield, dim, Kw, batch, out=None, col0=0):
    """OutterProductLayer('mat') with the kernel Kw [dim, P, dim] read in place: pair p's score goes to column
    col0 + p of ``out`` [B, ld] (default: a new [B, P])."""
    _require_cuda(x, Kw, out)
    if out is None:
        out = torch.empty((batch, nfield * (nfield - 1) // 2), dtype=torch.float32, device=x.device)
    _lib_call("pnn_outer_fwd", ptr(x), ldx, nfield, dim, ptr(Kw), ptr(out), out.stride(0), col0, batch, stream())
    return out


@_timed
def pnn_outer_bwd(g, ldg, gcol0, x, ldx, nfield, dim, Kw, batch, want_dx=True, want_dk=True):
    """-> (dx [B, nfield*dim] or None, dK [dim, P, dim] or None)."""
    _require_cuda(g, x, Kw)
    dev = x.device
    dx = torch.empty((batch, nfield * dim), dtype=torch.float32, device=dev) if want_dx else None
    dK = torch.empty(tuple(Kw.shape), dtype=torch.float32, device=dev) if want_dk else None
    nbytes = L.lib().b2ctr_pnn_outer_bwd_workspace_bytes(nfield, dim, batch) if want_dk else 0
    ws = workspace(nbytes, dev) if want_dk else None
    _lib_call("pnn_outer_bwd", ptr(g), ldg, gcol0, ptr(x), ldx, nfield, dim, ptr(Kw), ptr(dx), nfield * dim,
              ptr(dK), batch, ptr(ws), nbytes, stream())
    return dx, dK


REGULATE_MODES = {"copy": 0, "add": 1, "hadamard": 2, "attention": 3}   # b2ctr.h B2CTR_REGULATE_*
# limits of b2ctr_regulate_fwd / _bwd (include/b2ctr.h)
REGULATE_MAX_FIELDS, REGULATE_MAX_DIM = 1024, 256


def _2d(t):
    return (t.data_ptr(), t.stride(0)) if t is not None else (None, 0)


def _regulate_desc(mode, nfield, dim, batch, x, h, ax, ah, gates):
    """The operands of b2ctr_regulate_t: x / h / ax / ah 2-D [B, >= nfield*dim] views read in place (row pitch =
    stride(0)), ``gates`` [(g [nfield], inv_tau) or None] * 2."""
    _require_cuda(x, h, ax, ah)
    a = L.Regulate()
    a.mode, a.nfield, a.dim, a.batch = REGULATE_MODES[mode], nfield, dim, batch
    a.x, a.ldx = _2d(x)
    a.h, a.ldh = _2d(h)
    a.ax, a.ldax = _2d(ax)
    a.ah, a.ldah = _2d(ah)
    (g0, g1) = (list(gates) + [None, None])[:2]
    if g0 is not None:
        a.g0, a.inv_tau0 = g0[0].data_ptr(), float(g0[1])
    if g1 is not None:
        a.g1, a.inv_tau1 = g1[0].data_ptr(), float(g1[1])
    return a


def _window_of(a, name, out):
    """out = (tensor [B, ld], col0) or None -> the (ptr, ld, col) fields ``name`` of the descriptor."""
    if out is None:
        return
    t, col = out
    _require_cuda(t)
    setattr(a, name, t.data_ptr())
    setattr(a, "ld" + name, t.stride(0))
    setattr(a, name + "col", col)


@_timed
def regulate_fwd(mode, nfield, dim, batch, x, h=None, ax=None, ah=None, gates=(), u=None, y0=None, y1=None):
    """EDCN's bridge + gates in one pass (b2ctr_regulate_fwd): ``u`` / ``y0`` / ``y1`` are (buffer [B, ld], col0)
    windows to write v, v * gate0, v * gate1 into (None: not written)."""
    a = _regulate_desc(mode, nfield, dim, batch, x, h, ax, ah, gates)
    _window_of(a, "u", u)
    _window_of(a, "y0", y0)
    _window_of(a, "y1", y1)
    L.check(L.lib().b2ctr_regulate_fwd(C.byref(a), stream()), "regulate_fwd")


@_timed
def regulate_bwd(mode, nfield, dim, batch, x, h=None, ax=None, ah=None, gates=(), du=None, dy0=None, dy1=None,
                 want_dx=True, dx=None, dx_accumulate=False, want_dh=False, want_dax=False, want_dah=False,
                 want_dg=(False, False)):
    """-> (dx, dh, dax, dah, dg0, dg1) from the incoming gradients ``du`` / ``dy0`` / ``dy1`` ((buffer, col0) windows
    or None).  ``dx``: a 2-D view to write (or, with ``dx_accumulate``, add) x's gradient into; default a new
    [B, nfield*dim] tensor when ``want_dx``.  dh / dax / dah are new
    [B, nfield*dim] tensors when asked for, dg_k new [nfield] tensors."""
    a = _regulate_desc(mode, nfield, dim, batch, x, h, ax, ah, gates)
    _window_of(a, "u", du)
    _window_of(a, "y0", dy0)
    _window_of(a, "y1", dy1)
    dev, d = x.device, nfield * dim
    if not want_dx:
        dx = None
    elif dx is None:
        dx = torch.empty((batch, d), dtype=torch.float32, device=dev)
    _require_cuda(dx)
    dh, dax, dah = (torch.empty((batch, d), dtype=torch.float32, device=dev) if w else None
                    for w in (want_dh, want_dax, want_dah))
    dg = [torch.empty((nfield,), dtype=torch.float32, device=dev) if w else None for w in want_dg]
    a.dx, a.lddx = _2d(dx)
    a.dx_accumulate = int(bool(dx_accumulate))
    a.dh, a.lddh = _2d(dh)
    a.dax, a.lddax = _2d(dax)
    a.dah, a.lddah = _2d(dah)
    a.dg0 = dg[0].data_ptr() if dg[0] is not None else None
    a.dg1 = dg[1].data_ptr() if dg[1] is not None else None
    nbytes = L.lib().b2ctr_regulate_bwd_workspace_bytes(nfield, dim, batch) if any(w for w in want_dg) else 0
    ws = workspace(nbytes, dev)
    L.check(L.lib().b2ctr_regulate_bwd(C.byref(a), ptr(ws), nbytes, stream()), "regulate_bwd")
    return dx, dh, dax, dah, dg[0], dg[1]



# limits of b2ctr_conv_stack_fwd / _bwd (include/b2ctr.h)
CONV_MAX_ROWS, CONV_MAX_CHANNELS, CONV_MAX_WIDTH, CONV_SMEM_BYTES = 64, 16, 32, 224 * 1024


def conv_stack_check(rows, channels, stages):
    """Raise ValueError naming the limit of b2ctr_conv_stack that ``stages`` on a [rows, channels] column breaks.
    ``stages``: ("conv", width, filters) or ("kmax", k) tuples (extra entries ignored).  Returns the last map's
    (rows, channels)."""
    if not 1 <= len(stages) <= L.CONV_STACK_MAX_STAGES:
        raise ValueError("the convolution stack supports 1 to %d stages (got %d)"
                         % (L.CONV_STACK_MAX_STAGES, len(stages)))
    if not 1 <= rows <= CONV_MAX_ROWS:
        raise ValueError("the convolution stack supports 1 to %d rows (CONV_MAX_ROWS), got %d" % (CONV_MAX_ROWS, rows))
    if not 1 <= channels <= CONV_MAX_CHANNELS:
        raise ValueError("the convolution stack supports 1 to %d channels (CONV_MAX_CHANNELS), got %d"
                         % (CONV_MAX_CHANNELS, channels))
    maps = [rows * channels]
    nw = 0
    for st in stages:
        if st[0] == "conv":
            width, filters = st[1], st[2]
            if not 1 <= width <= CONV_MAX_WIDTH:
                raise ValueError("Conv2D supports kernel widths 1 to %d (CONV_MAX_WIDTH), got %d"
                                 % (CONV_MAX_WIDTH, width))
            if not 1 <= filters <= CONV_MAX_CHANNELS:
                raise ValueError("Conv2D supports 1 to %d filters (CONV_MAX_CHANNELS), got %d"
                                 % (CONV_MAX_CHANNELS, filters))
            nw += width * channels * filters + filters
            channels = filters
            maps.append(rows * channels)
        else:
            if not 1 <= st[1] <= rows:
                raise ValueError("k must be in 1 ~ %d,now k is %d" % (rows, st[1]))
            rows = st[1]
            maps += [rows * channels, rows * channels]
    smem = 4 * (2 * nw + 32 * (sum(maps) + 2 * max(maps)))
    if smem > CONV_SMEM_BYTES:
        raise ValueError("the convolution stack needs %d bytes of shared memory per 32 columns, above its %d-byte "
                         "limit (CONV_SMEM_BYTES): fewer rows or channels" % (smem, CONV_SMEM_BYTES))
    return rows, channels


def _conv_desc(stages, x, rows, dim, channels, batch, out):
    """b2ctr_conv_stack_t over x (2-D [B, >= rows*dim*channels] view read in place, pitch stride(0)) and out (the
    forward output or the backward's incoming gradient, the same kind of view).  ``stages``: ("conv", width,
    filters, act, kernel, bias or None) or ("kmax", k)."""
    _require_cuda(x, out)
    a = L.ConvStack()
    a.struct_size = C.sizeof(L.ConvStack)
    a.nstage, a.rows, a.dim, a.channels, a.batch = len(stages), rows, dim, channels, batch
    a.x, a.ldx = x.data_ptr(), x.stride(0)
    a.out, a.ldout = out.data_ptr(), out.stride(0)
    for i, st in enumerate(stages):
        d = a.stage[i]
        if st[0] == "conv":
            _, width, filters, act, kernel, bias = st
            _require_cuda(kernel, bias)
            d.kind, d.width, d.filters, d.act = L.CONV_STAGE_CONV, width, filters, L.ACT_BY_NAME[act]
            d.kernel = kernel.data_ptr()
            d.bias = bias.data_ptr() if bias is not None else None
        else:
            d.kind, d.k = L.CONV_STAGE_KMAX, st[1]
    return a


@_timed
def conv_stack_fwd(stages, x, rows, dim, channels, batch, out):
    """CCPM's conv / k-max stack per (sample, e) column in one launch (b2ctr_conv_stack_fwd): x [B, rows, dim,
    channels] read in place, the last map written in Flatten order into ``out`` (a 2-D view)."""
    a = _conv_desc(stages, x, rows, dim, channels, batch, out)
    L.check(L.lib().b2ctr_conv_stack_fwd(C.byref(a), stream()), "conv_stack_fwd")
    return out


@_timed
def conv_stack_bwd(stages, x, rows, dim, channels, batch, dout, dx=None, dx_accumulate=False, want_dw=()):
    """Recompute the stack and take its gradient (b2ctr_conv_stack_bwd): ``dx`` a 2-D view to write (or add) x's
    gradient into, or None; ``want_dw`` per conv stage whether its (dkernel, dbias) are wanted.  Returns the list of
    (dkernel, dbias) per stage (None for k-max stages or when not wanted)."""
    a = _conv_desc(stages, x, rows, dim, channels, batch, dout)
    if dx is not None:
        _require_cuda(dx)
        a.dx, a.lddx, a.dx_accumulate = dx.data_ptr(), dx.stride(0), int(bool(dx_accumulate))
    dws = []
    for i, st in enumerate(stages):
        if st[0] == "conv" and (want_dw[i] if i < len(want_dw) else False):
            dk = torch.empty(tuple(st[4].shape), dtype=torch.float32, device=x.device)
            db = torch.empty((st[2],), dtype=torch.float32, device=x.device) if st[5] is not None else None
            a.stage[i].dkernel = dk.data_ptr()
            a.stage[i].dbias = db.data_ptr() if db is not None else None
            dws.append((dk, db))
        else:
            dws.append(None)
    nbytes = L.lib().b2ctr_conv_stack_bwd_workspace_bytes(C.byref(a)) if any(d is not None for d in dws) else 0
    ws = workspace(nbytes, x.device)
    L.check(L.lib().b2ctr_conv_stack_bwd(C.byref(a), ptr(ws), nbytes, stream()), "conv_stack_bwd")
    return dws

# limits of b2ctr_field_wise_bi_fwd / _bwd (include/b2ctr.h)
FWBI_MAX_DIM = 256


def field_wise_bi_check(nfield, ngroup, dim):
    """Raise ValueError naming the limit of b2ctr_field_wise_bi that nfield fields in ngroup groups of dim
    coordinates break."""
    if not 2 <= ngroup <= L.FWBI_MAX_GROUPS:
        raise ValueError("FieldWiseBiInteraction supports 2 to %d groups (FWBI_MAX_GROUPS), got %d"
                         % (L.FWBI_MAX_GROUPS, ngroup))
    if not ngroup <= nfield <= L.FWBI_MAX_FIELDS:
        raise ValueError("FieldWiseBiInteraction supports at most %d fields in all (FWBI_MAX_FIELDS), got %d"
                         % (L.FWBI_MAX_FIELDS, nfield))
    if not 1 <= dim <= FWBI_MAX_DIM:
        raise ValueError("FieldWiseBiInteraction supports embedding_size 1 to %d (FWBI_MAX_DIM), got %d"
                         % (FWBI_MAX_DIM, dim))


def _fwbi_desc(x, cols, groups, ngroup, dim, batch, kernel_mf, kernel_fm, bias_mf, bias_fm, out, outcol):
    """b2ctr_field_wise_bi_t: field f is the [dim] row at column cols[f] of x (a 2-D [B, ld] view read in place,
    pitch stride(0)) in group groups[f]; ``out`` a 2-D view whose columns [outcol, outcol + dim) are h (forward)
    or dh (backward)."""
    _require_cuda(x, kernel_mf, kernel_fm, bias_mf, bias_fm, out)
    a = L.FieldWiseBi()
    a.struct_size = C.sizeof(L.FieldWiseBi)
    a.nfield, a.ngroup, a.dim, a.batch = len(cols), ngroup, dim, batch
    if len(cols) > L.FWBI_MAX_FIELDS:
        raise ValueError("FieldWiseBiInteraction supports at most %d fields in all (FWBI_MAX_FIELDS), got %d"
                         % (L.FWBI_MAX_FIELDS, len(cols)))
    for f, (c, g) in enumerate(zip(cols, groups)):
        a.col[f], a.group[f] = c, g
    a.x, a.ldx = x.data_ptr(), x.stride(0)
    a.kernel_mf, a.kernel_fm = kernel_mf.data_ptr(), kernel_fm.data_ptr()
    a.bias_mf = bias_mf.data_ptr() if bias_mf is not None else None
    a.bias_fm = bias_fm.data_ptr() if bias_fm is not None else None
    a.out, a.ldout, a.outcol = out.data_ptr(), out.stride(0), outcol
    return a


@_timed
def field_wise_bi_fwd(x, cols, groups, ngroup, dim, batch, kernel_mf, kernel_fm, bias_mf, bias_fm, out, outcol=0):
    """FLEN's FieldWiseBiInteraction in one launch (b2ctr_field_wise_bi_fwd): reads the fields in place and writes
    only h into the columns [outcol, outcol + dim) of ``out``."""
    a = _fwbi_desc(x, cols, groups, ngroup, dim, batch, kernel_mf, kernel_fm, bias_mf, bias_fm, out, outcol)
    L.check(L.lib().b2ctr_field_wise_bi_fwd(C.byref(a), stream()), "field_wise_bi_fwd")
    return out


@_timed
def field_wise_bi_bwd(x, cols, groups, ngroup, dim, batch, kernel_mf, kernel_fm, bias_mf, bias_fm, dout, doutcol=0,
                      dx=None, dx_accumulate=False, want_dkernel=(False, False), want_dbias=(False, False)):
    """Recompute the forward and take its gradient (b2ctr_field_wise_bi_bwd): ``dx`` a 2-D view whose columns
    cols[f] take (or, with ``dx_accumulate``, add) field f's gradient, or None.  Returns (dkernel_mf [P, 1],
    dkernel_fm [G, 1], dbias_mf [dim], dbias_fm [dim]), None where not wanted."""
    a = _fwbi_desc(x, cols, groups, ngroup, dim, batch, kernel_mf, kernel_fm, bias_mf, bias_fm, dout, doutcol)
    if dx is not None:
        _require_cuda(dx)
        a.dx, a.lddx, a.dx_accumulate = dx.data_ptr(), dx.stride(0), int(bool(dx_accumulate))
    dev = x.device
    shapes = ((ngroup * (ngroup - 1) // 2, 1), (ngroup, 1), (dim,), (dim,))
    res = [torch.empty(sh, dtype=torch.float32, device=dev) if w else None
           for sh, w in zip(shapes, tuple(want_dkernel) + tuple(want_dbias))]
    a.dkernel_mf, a.dkernel_fm, a.dbias_mf, a.dbias_fm = [t.data_ptr() if t is not None else None for t in res]
    nbytes = (L.lib().b2ctr_field_wise_bi_bwd_workspace_bytes(C.byref(a))
              if any(t is not None for t in res) else 0)
    ws = workspace(nbytes, dev)
    L.check(L.lib().b2ctr_field_wise_bi_bwd(C.byref(a), ptr(ws), nbytes, stream()), "field_wise_bi_bwd")
    return tuple(res)


@_timed
def din_att_input_fwd(q, ldq, keys, ldk, batch, T, E):
    out = torch.empty((batch, T, 4 * E), dtype=torch.float32, device=q.device)
    _lib_call("din_att_input_fwd", ptr(q), ldq, ptr(keys), ldk, ptr(out), batch, T, E, stream())
    return out


@_timed
def din_att_input_bwd(q, ldq, keys, ldk, g, batch, T, E):
    dq = torch.empty((batch, 1, E), dtype=torch.float32, device=q.device)
    dk = torch.empty((batch, T, E), dtype=torch.float32, device=q.device)
    _lib_call("din_att_input_bwd", ptr(q), ldq, ptr(keys), ldk, ptr(g), ptr(dq), ptr(dk), batch, T, E, stream())
    return dq, dk


@_timed
def din_pool_fwd(score, keys, ldk, mask, batch, T, E, weight_norm, return_score):
    w = torch.empty((batch, T), dtype=torch.float32, device=score.device)
    out = torch.empty((batch, 1, T if return_score else E), dtype=torch.float32, device=score.device)
    _lib_call("din_pool_fwd", ptr(score), ptr(keys), ldk, ptr(mask), ptr(w), ptr(out), batch, T, E,
              int(weight_norm), int(return_score), stream())
    return out, w


@_timed
def din_pool_bwd(w, keys, ldk, mask, dout, batch, T, E, weight_norm, return_score, want_dkeys=True):
    dscore = torch.empty((batch, T, 1), dtype=torch.float32, device=w.device)
    dkeys = torch.empty((batch, T, E), dtype=torch.float32, device=w.device) if (want_dkeys and not return_score) \
        else None
    _lib_call("din_pool_bwd", ptr(w), ptr(keys), ldk, ptr(mask), ptr(dout), ptr(dscore), ptr(dkeys), batch, T, E,
              int(weight_norm), int(return_score), stream())
    return dscore, dkeys


@_timed
def seqpool_fwd(x, mask, length, batch, T, E, mode):
    out = torch.empty((batch, 1, E), dtype=torch.float32, device=x.device)
    _lib_call("seqpool_fwd", ptr(x), ptr(mask), ptr(length), ptr(out), batch, T, E, mode, stream())
    return out


@_timed
def seqpool_bwd(x, mask, length, dout, batch, T, E, mode):
    dx = torch.empty((batch, T, E), dtype=torch.float32, device=x.device)
    _lib_call("seqpool_bwd", ptr(x), ptr(mask), ptr(length), ptr(dout), ptr(dx), batch, T, E, mode, stream())
    return dx


@_timed
def seqweight(w, mask, length, batch, T, normalize):
    wt = torch.empty((batch, T), dtype=torch.float32, device=w.device)
    _lib_call("seqweight", ptr(w), ptr(mask), ptr(length), ptr(wt), batch, T, int(normalize), stream())
    return wt


@_timed
def seqscale(x, wt, rows, E):
    out = torch.empty_like(x)
    _lib_call("seqscale", ptr(x), ptr(wt), ptr(out), rows, E, stream())
    return out


@_timed
def colstats(x, ld, m, n):
    stats = torch.empty((2, n), dtype=torch.float32, device=x.device)
    nbytes = L.lib().b2ctr_colstats_workspace_bytes(m, n)
    ws = workspace(nbytes, x.device)
    _lib_call("colstats", ptr(x), ld, m, n, ptr(stats), ptr(ws), nbytes, stream())
    return stats


@_timed
def moving_update(moving, batch_stat, momentum):
    _lib_call("moving_update", ptr(moving), ptr(batch_stat), momentum, moving.numel(), stream())


@_timed
def bn_apply(x, mean, var, gamma, beta, m, n, eps):
    y = torch.empty_like(x)
    _lib_call("bn_apply", ptr(x), ptr(mean), ptr(var), ptr(gamma), ptr(beta), ptr(y), m, n, eps, stream())
    return y


@_timed
def bn_bwd(x, mean, var, gamma, dy, m, n, eps, training):
    dx = torch.empty_like(x)
    dgamma = torch.empty((n,), dtype=torch.float32, device=x.device)
    dbeta = torch.empty((n,), dtype=torch.float32, device=x.device)
    nbytes = L.lib().b2ctr_colstats_workspace_bytes(m, n)
    ws = workspace(nbytes, x.device)
    _lib_call("bn_bwd", ptr(x), ptr(mean), ptr(var), ptr(gamma), ptr(dy), ptr(dx), ptr(dgamma), ptr(dbeta), m, n,
              eps, int(training), ptr(ws), nbytes, stream())
    return dx, dgamma, dbeta


@_timed
def dice_fwd(x, mean, var, alpha, m, n, eps):
    y = torch.empty_like(x)
    _lib_call("dice_fwd", ptr(x), ptr(mean), ptr(var), ptr(alpha), ptr(y), m, n, eps, stream())
    return y


@_timed
def dice_bwd(x, mean, var, alpha, dy, m, n, eps, training):
    dx = torch.empty_like(x)
    dalpha = torch.empty((n,), dtype=torch.float32, device=x.device)
    nbytes = L.lib().b2ctr_dice_bwd_workspace_bytes(m, n)
    ws = workspace(nbytes, x.device)
    _lib_call("dice_bwd", ptr(x), ptr(mean), ptr(var), ptr(alpha), ptr(dy), ptr(dx), ptr(dalpha), m, n, eps,
              int(training), ptr(ws), nbytes, stream())
    return dx, dalpha


@_timed
def dropout(x, rate, seed):
    y = torch.empty_like(x)
    _lib_call("dropout", ptr(x), ptr(y), x.numel(), rate, seed & 0xFFFFFFFFFFFFFFFF, stream())
    return y


def _mha_desc(q, ldq, k, ldk, v, ldv, batch, T, heads, d, scale, blinding, rate, seed, stats, qlen, klen, qmask,
              kmask):
    a = L.Mha()
    a.q, a.ldq, a.k, a.ldk, a.v, a.ldv = q.data_ptr(), ldq, k.data_ptr(), ldk, v.data_ptr(), ldv
    a.stats = stats.data_ptr()
    a.qlen, a.klen = (qlen.data_ptr() if qlen is not None else None), (klen.data_ptr() if klen is not None else None)
    a.qmask = qmask.data_ptr() if qmask is not None else None
    a.kmask = kmask.data_ptr() if kmask is not None else None
    a.batch, a.T, a.heads, a.d = batch, T, heads, d
    a.scale, a.blinding, a.dropout_rate, a.seed = scale, int(blinding), rate, seed & 0xFFFFFFFFFFFFFFFF
    return a


@_timed
def mha_fwd(q, ldq, k, ldk, v, ldv, batch, T, heads, d, scale, blinding=False, rate=0.0, seed=0, res=None, ldr=0,
            qlen=None, klen=None, qmask=None, kmask=None):
    """Masked multi-head attention over rows b*T + t of q / k / v (row pitches ld*) -> (out [B*T, heads*d],
    softmax statistics [B, heads, T, 2]).  Validity from int32 lengths [B] or uint8 masks [B, T]."""
    _require_cuda(q, k, v, res)
    out = torch.empty((batch * T, heads * d), dtype=torch.float32, device=q.device)
    stats = torch.empty((batch, heads, T, 2), dtype=torch.float32, device=q.device)
    a = _mha_desc(q, ldq, k, ldk, v, ldv, batch, T, heads, d, scale, blinding, rate, seed, stats, qlen, klen, qmask,
                  kmask)
    a.res, a.ldr = (res.data_ptr() if res is not None else None), ldr
    a.out, a.ldo = out.data_ptr(), heads * d
    L.check(L.lib().b2ctr_mha_fwd(C.byref(a), stream()), "mha_fwd")
    return out, stats


@_timed
def mha_bwd(dout, lddo, q, ldq, k, ldk, v, ldv, stats, batch, T, heads, d, scale, blinding=False, rate=0.0, seed=0,
            qlen=None, klen=None, qmask=None, kmask=None):
    """-> (dq, dk, dv), each [B*T, heads*d]."""
    _require_cuda(dout, q, k, v, stats)
    w = heads * d
    dq, dk, dv = (torch.empty((batch * T, w), dtype=torch.float32, device=q.device) for _ in range(3))
    a = _mha_desc(q, ldq, k, ldk, v, ldv, batch, T, heads, d, scale, blinding, rate, seed, stats, qlen, klen, qmask,
                  kmask)
    a.dout, a.lddo = dout.data_ptr(), lddo
    a.dq, a.lddq, a.dk, a.lddk, a.dv, a.lddv = dq.data_ptr(), w, dk.data_ptr(), w, dv.data_ptr(), w
    L.check(L.lib().b2ctr_mha_bwd(C.byref(a), stream()), "mha_bwd")
    return dq, dk, dv


@_timed
def layernorm_fwd(a, lda, b, ldb, gamma, beta, rows, n, eps):
    """LayerNormalization of a (+ b) over rows of n columns -> (y [rows, n], stats (mean, rstd) [rows, 2])."""
    _require_cuda(a, b, gamma, beta)
    y = torch.empty((rows, n), dtype=torch.float32, device=a.device)
    stats = torch.empty((rows, 2), dtype=torch.float32, device=a.device)
    _lib_call("layernorm_fwd", ptr(a), lda, ptr(b), ldb, ptr(gamma), ptr(beta), ptr(y), n, ptr(stats), rows, n, eps,
              stream())
    return y, stats


@_timed
def layernorm_bwd(a, lda, b, ldb, gamma, stats, dy, rows, n, want_dgamma=True, want_dbeta=True):
    """-> (dx [rows, n], dgamma [n] | None, dbeta [n] | None)."""
    _require_cuda(a, b, gamma, stats, dy)
    dev = a.device
    dx = torch.empty((rows, n), dtype=torch.float32, device=dev)
    dgamma = torch.empty((n,), dtype=torch.float32, device=dev) if want_dgamma else None
    dbeta = torch.empty((n,), dtype=torch.float32, device=dev) if want_dbeta else None
    nbytes = L.lib().b2ctr_layernorm_bwd_workspace_bytes(rows, n)
    ws = workspace(nbytes, dev)
    _lib_call("layernorm_bwd", ptr(a), lda, ptr(b), ldb, ptr(gamma), ptr(stats), ptr(dy), dy.stride(0), ptr(dx), n,
              ptr(dgamma), ptr(dbeta), rows, n, ptr(ws), nbytes, stream())
    return dx, dgamma, dbeta


# ---- row-sharded embedding exchange (device side) ----------------------------------------------------
@_timed
def shard_bucketize(feats, batch, world):
    """-> (counts int32 [world], slot int64 [B*F]) for the lookups described by feats[f].idx."""
    dev = torch.device("cuda", torch.cuda.current_device())
    counts = torch.empty((world,), dtype=torch.int32, device=dev)
    fill(counts.view(torch.float32), 0.0)
    slot = torch.empty((batch * len(feats),), dtype=torch.int64, device=dev)
    arr = _feat_array(feats)
    _lib_call("shard_bucketize", arr, len(feats), batch, world, ptr(counts), ptr(slot), stream())
    return counts, slot


@_timed
def shard_fill(feats, batch, world, counts, slot):
    dev = counts.device
    n = batch * len(feats)
    keys = torch.empty((n,), dtype=torch.int64, device=dev)
    pos = torch.empty((batch, len(feats)), dtype=torch.int32, device=dev)
    arr = _feat_array(feats)
    _lib_call("shard_fill", arr, len(feats), batch, world, ptr(counts), ptr(slot), ptr(keys), ptr(pos), stream())
    return keys, pos


def _ptr_array(tensors):
    return (C.c_void_p * len(tensors))(*[t.data_ptr() if t is not None else None for t in tensors])


@_timed
def shard_gather_rows(tables, lin_tables, dim, keys, n):
    dev = keys.device
    rows = torch.empty((max(n, 1), dim), dtype=torch.float32, device=dev)
    lin = torch.empty((max(n, 1),), dtype=torch.float32, device=dev) if lin_tables is not None else None
    _lib_call("shard_gather_rows", _ptr_array(tables), _ptr_array(lin_tables) if lin_tables is not None else None,
              len(tables), dim, ptr(keys), n, ptr(rows), ptr(lin), stream())
    return rows, lin


@_timed
def shard_scatter_rows(tables, lin_tables, dim, keys, n, grows, glin, scale, lin_scale):
    _lib_call("shard_scatter_rows", _ptr_array(tables), _ptr_array(lin_tables) if lin_tables is not None else None,
              len(tables), dim, ptr(keys), n, ptr(grows), ptr(glin), scale, lin_scale, stream())
