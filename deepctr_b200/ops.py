"""Differentiable ops on ``engine.Var``: each launches libb2ctr kernels for the forward and pushes a
closure on the active tape that launches the backward kernels.  No torch arithmetic anywhere.
"""
import ctypes

import numpy as np
import torch

from . import _lib as L
from . import kernels as K
from . import engine as E

# precision mode used by every dense GEMM (DNN / attention MLP / projections); see DESIGN.md section 5.
# Default: split-bf16 on the wgmma tensor cores (three bf16 MMAs per product, fp32 accumulation; relative
# error ~2^-16, inside the 1e-4 logit tolerance of the parity tests); 'fp32' selects the exact FFMA GEMM.
GEMM_PRECISION = L.GEMM_BF16X3


# bumped by ops whose kernels take per-step by-value state (dropout seeds) or that need the host (string
# hashing): a model that ran one of them is never replayed as a CUDA graph (engine.Model._graph_eligible)
UNCAPTURABLE = 0


def mark_uncapturable():
    global UNCAPTURABLE
    UNCAPTURABLE += 1


def set_gemm_precision(mode):
    """'fp32' (exact FFMA) or 'bf16x3' (wgmma split-bf16, ~2^-17 relative)."""
    global GEMM_PRECISION
    GEMM_PRECISION = {"fp32": L.GEMM_FP32, "bf16x3": L.GEMM_BF16X3}[mode]


def _empty(shape, like):
    return torch.empty(shape, dtype=torch.float32, device=like.device)


def _split_k(m_out, n_out, kred):
    """wgrad-style GEMMs reduce over the batch: split K until the output, counted in 256 x 256 blocks, times the
    slices makes about 74 blocks (at least 1024 rows per slice).  That is about 296 of the persistent kernel's
    128 x 128 tiles, a little over two per SM on the 132 SMs of an H100 (845 x 256: 4 blocks, 18 slices)."""
    if kred < 4096:
        return 1
    if n_out <= 8:
        # skinny wgrad (the [*, 1] projections, CrossNet's w): an HBM stream over the batch handled by
        # skinny_tn_kernel, one CTA per (64-column block, K slice) - slices of ~256 rows, up to 4 CTAs per SM
        # (64 slices of 1024 rows left 57 % of the SMs idle: 86 us for a 16 MB read, ncu r2_launches_c2.csv)
        blocks = (m_out + 63) // 64
        return int(max(1, min(592 // blocks, kred // 256)))
    tiles = ((m_out + 255) // 256) * ((n_out + 255) // 256)
    return int(max(1, min(74 // tiles if tiles <= 74 else 1, kred // 1024)))


def _as2d(x):
    t2, ld = x.as2d()
    if t2 is None:
        t = E.contiguous(x)
        t2 = t.reshape(-1, t.shape[-1])
        ld = t2.stride(0)
    return t2, ld


# ---- GEMM based --------------------------------------------------------------------------------
def _planes_of(var, t2):
    """bf16 hi/lo planes of a Var's 2-D view, split once per step and shared by every GEMM that reads it
    (forward of each consumer + the wgrad GEMMs)."""
    base = var.base
    if base is not None and hasattr(base.owner, "lookup_planes"):
        planes = base.owner.lookup_planes(var, t2)     # the fused embedding gather wrote them
        if planes is not None:
            return planes
    key = (t2.data_ptr(), tuple(t2.shape), t2.stride(0))
    if var.planes is None or var.planes[0] != key:
        var.planes = (key, K.split_planes(t2))
    return var.planes[1]


class _Layer(object):
    """What the backward of one act(x @ w + b) GEMM layer needs: the operands, their planes and the precision."""
    __slots__ = ("x2", "m", "kdim", "n", "wd", "prec", "reuse", "xp", "wp")


def _dense_fwd(x, w, b, act):
    """act(x @ w + b) over the last axis of x as one GEMM, bias and activation in its epilogue; returns (y [m, n],
    the _Layer its backward reads)."""
    st = _Layer()
    st.x2, _ = _as2d(x)
    st.m, st.kdim = st.x2.shape
    st.n = w.shape[1]
    st.wd = w.materialize() if isinstance(w, E.Weight) else w.data
    bd = (b.materialize() if isinstance(b, E.Weight) else b.data) if b is not None else None
    # BF16X3: operands are split into bf16 planes once and the planes are reused by forward/dgrad/wgrad
    # skinny layers (the final [*, 1] projection) are GEMVs: exact-fp32 FFMA path, no tensor-core staging
    st.prec = GEMM_PRECISION if min(st.n, st.kdim) >= 16 else L.GEMM_FP32
    st.reuse = st.prec == L.GEMM_BF16X3 and st.m >= 128
    st.xp = _planes_of(x, st.x2) if st.reuse else None
    st.wp = K.split_planes(st.wd) if st.reuse else None
    y = K.gemm(st.x2, st.wd, bias=bd, act=act, precision=st.prec, m=st.m, n=st.n, k=st.kdim, a_planes=st.xp,
               b_planes=st.wp)
    return y, st


def _dense_grads(x, w, st, dz, dzp):
    """dx = dz w^T and dw = x^T dz of a _dense_fwd layer, added to x's and w's gradients.  dz may be None when its
    planes dzp are given."""
    m, kdim, n, prec = st.m, st.kdim, st.n, st.prec
    if x.requires_grad:
        base = x.base
        if (base is not None and x.col0 == 0 and x.ncols != -1 and base.data.dim() == 2
                and base.data.shape[0] == m and x.ncols == kdim):
            # x is the leading window of a K-padded buffer: write dx with the same ld so that
            # the buffer's gradient is adopted without a copy
            ld = base.data.stride(0)
            buf = _empty((m, ld), base.data)
            dxw = buf[:, :kdim]
            K.gemm(dz, st.wd, c=dxw, trans_b=True, precision=prec, m=m, n=kdim, k=n, a_planes=dzp,
                   b_planes=st.wp)
            E.add_grad(x, dxw)
        else:
            dx = K.gemm(dz, st.wd, trans_b=True, precision=prec, m=m, n=kdim, k=n, a_planes=dzp,
                        b_planes=st.wp)
            E.add_grad(x, dx.reshape(x.data.shape))
    if w.requires_grad:
        dw = K.gemm(st.x2, dz, trans_a=True, precision=prec, split_k=_split_k(kdim, n, m),
                    m=kdim, n=n, k=m, a_planes=st.xp, b_planes=dzp)
        E.add_grad(w, dw)


def dense(x, w, b=None, activation=None):
    """y = act(x @ w + b) over the last axis (tf.tensordot(x, w, axes=(-1, 0)) + bias_add)."""
    act = L.ACT_BY_NAME.get(activation, None)
    fused_act = act if act is not None else L.ACT_NONE
    y, st = _dense_fwd(x, w, b, fused_act)
    m, n = st.m, st.n
    out = E.Var(y.reshape(tuple(x.data.shape[:-1]) + (n,)))
    if act is None and activation is not None:
        raise ValueError("activation %r cannot be fused into dense(); apply it as a layer" % activation)

    def bwd(grads):
        dy = grads[0].reshape(m, n)
        if not dy.is_contiguous():
            dy = dy.contiguous()
        need_db = b is not None and b.requires_grad
        need_planes = st.reuse and (x.requires_grad or w.requires_grad)
        dzp = None
        if fused_act != L.ACT_NONE or need_db:
            if need_planes and fused_act != L.ACT_NONE and dy.stride(0) % 4 == 0 and K.planes_fusable(m, n):
                # the dgrad and wgrad below read only the planes (n >= 64 here): dz itself is never written
                dz, db, dzp = K.bias_act_bwd(dy, y, fused_act, want_dz=False, want_dbias=need_db, want_planes=True)
            else:
                dz, db = K.bias_act_bwd(dy, y, fused_act, want_dz=fused_act != L.ACT_NONE, want_dbias=need_db)
                if dz is None:
                    dz = dy
        else:
            dz, db = dy, None
        if need_planes and dzp is None:
            dzp = K.split_planes(dz)
        _dense_grads(x, w, st, dz, dzp)
        if need_db:
            E.add_grad(b, db)

    E.record([out], [x, w, b], bwd)
    return out


def mlp_fusable(x, widths):
    """ops.mlp runs this relu tower: split-bf16 GEMMs, layer 0 on operand planes (at least 128 rows, both of its
    dimensions at least 16) and fused kernels for the widths after it."""
    m = int(np.prod(x.data.shape[:-1]))
    return (GEMM_PRECISION == L.GEMM_BF16X3 and len(widths) >= 2 and m >= 128 and x.data.shape[-1] >= 16
            and widths[0] >= 16 and L.lib().b2ctr_mlp_relu_supported((ctypes.c_int32 * len(widths))(*widths),
                                                                     len(widths)) == 1)


def mlp(x, kernels, biases):
    """A relu DNN tower, y_i = relu(y_{i-1} W_i + b_i), as one tape node (mlp_fusable must hold): layer 0 is
    dense()'s GEMM, the layers after it one fused forward kernel; the backward runs one fused kernel for every
    layer's bias and activation gradient, then the split-K weight-gradient GEMMs on the planes it wrote and
    layer 0's dgrad."""
    y0, st = _dense_fwd(x, kernels[0], biases[0], L.ACT_RELU)
    ws = [w.materialize() if isinstance(w, E.Weight) else w.data for w in kernels[1:]]
    bs = [b.materialize() if isinstance(b, E.Weight) else b.data for b in biases[1:]]
    planes, y = K.mlp_relu_fwd(y0, ws, bs)
    out = E.Var(y.reshape(tuple(x.data.shape[:-1]) + (y.shape[1],)))

    def bwd(grads):
        dzp, db = K.mlp_relu_bwd(grads[0].reshape(y.shape), y, y0, planes, ws)
        _dense_grads(x, kernels[0], st, None, dzp[0])
        m = st.m
        for i in range(1, len(kernels)):
            if kernels[i].requires_grad:
                kdim, n = ws[i - 1].shape
                dw = K.gemm(None, None, trans_a=True, precision=L.GEMM_BF16X3, split_k=_split_k(kdim, n, m),
                            m=kdim, n=n, k=m, a_planes=planes[i - 1], b_planes=dzp[i])
                E.add_grad(kernels[i], dw)
        for bias, g in zip(biases, db):
            E.add_grad(bias, g)

    E.record([out], [x] + list(kernels) + list(biases), bwd)
    return out


def activation(x, name):
    act = L.ACT_BY_NAME[name]
    if act == L.ACT_NONE:
        return x
    xt = E.contiguous(x)
    y = K.act_fwd(xt, act)
    out = E.Var(y)

    def bwd(grads):
        dz, _ = K.bias_act_bwd(grads[0].reshape(-1, y.shape[-1]).contiguous(), y.reshape(-1, y.shape[-1]),
                               act, want_dz=True, want_dbias=False)
        E.add_grad(x, dz.reshape(x.data.shape))

    E.record([out], [x], bwd)
    return out


# ---- shape plumbing (zero-copy whenever the operands alias one buffer) --------------------------
def _window(base, col0, ncols, shape, mask=None):
    bt = base.data
    b = bt.shape[0]
    dense_strides = []
    acc = 1
    for s in reversed(shape[1:]):
        dense_strides.append(acc)
        acc *= s
    dense_strides = list(reversed(dense_strides))
    data = bt.as_strided((b,) + tuple(shape[1:]), (bt.stride(0),) + tuple(dense_strides),
                         bt.storage_offset() + col0)
    return E.Var(data, requires_grad=base.requires_grad, mask=mask, base=base, col0=col0, ncols=ncols,
                 owner=base.owner)


def flatten(x):
    b = x.data.shape[0]
    w = int(np.prod(x.data.shape[1:]))
    if x.base is not None and x.ncols != -1:
        return _window(x.base, x.col0, x.ncols, (b, w))
    t = E.contiguous(x)
    out = E.Var(t.reshape(b, w))
    out.base, out.col0, out.ncols = x if x.base is None else x.base, 0, -1
    out.requires_grad = x.requires_grad
    return out


def reshape(x, shape):
    """Per-sample reshape (batch dim kept)."""
    b = x.data.shape[0]
    shape = (b,) + tuple(shape[1:])
    if x.base is not None and x.ncols != -1:
        return _window(x.base, x.col0, x.ncols, shape, x.mask)
    t = E.contiguous(x)
    out = E.Var(t.reshape(shape), mask=x.mask)
    out.base, out.col0, out.ncols = x if x.base is None else x.base, 0, -1
    out.requires_grad = x.requires_grad
    return out


def _flat_concat_ok(shapes, axis):
    nd = len(shapes[0])
    ax = axis if axis >= 0 else nd + axis
    return ax, all(all(s[d] == 1 for d in range(1, ax)) for s in shapes)


def concat(xs, axis=-1):
    xs = list(xs)
    if len(xs) == 1:
        return xs[0]
    shapes = [tuple(v.shape) for v in xs]
    ax, flat_ok = _flat_concat_ok(shapes, axis)
    out_shape = list(shapes[0])
    out_shape[ax] = sum(s[ax] for s in shapes)
    b = shapes[0][0]
    widths = [int(np.prod(s[1:])) for s in shapes]
    if flat_ok:
        # zero-copy: adjacent windows of the same buffer, in order
        base = xs[0].base
        if base is not None and xs[0].ncols != -1:
            col = xs[0].col0
            ok = True
            for v, w in zip(xs, widths):
                if v.base is not base or v.ncols == -1 or v.col0 != col or v.ncols != w:
                    ok = False
                    break
                col += w
            if ok and base.data is None:     # virtual buffer (fused away): stay virtual
                return E.Var(None, base=base, col0=xs[0].col0, ncols=col - xs[0].col0, owner=base.owner,
                             vshape=tuple(out_shape))
            if ok:
                return _window(base, xs[0].col0, col - xs[0].col0, tuple(out_shape))
    if any(v.data is None for v in xs):
        raise L.B2ctrError("a fused-away (virtual) embedding output reached a layer that needs its values")
    if flat_ok:
        # per-sample flat concatenation of non-adjacent windows: strided 2-D copies, no densifying pass
        out = _empty((b, sum(widths)), xs[0].data)
        col = 0
        for v, w in zip(xs, widths):
            src, ld = v.flat2d()
            if src is None:
                src = E.contiguous(v).reshape(b, w)
                ld = w
            K.copy2d(src, ld, out, out.stride(0), b, w, dst_off=col)
            col += w
        res = E.Var(out.reshape(out_shape))

        def bwd(grads):
            g = grads[0].reshape(b, -1)
            c = 0
            for v, w in zip(xs, widths):
                if v.requires_grad:
                    gv = _empty((b, w), g)
                    K.copy2d(g, g.stride(0), gv, w, b, w, src_off=c)
                    E.add_grad(v, gv.reshape(v.data.shape))
                c += w

        E.record([res], xs, bwd)
        return res
    # general case: concatenate along `ax` with non-unit leading dims -> rows = prod(dims < ax)
    lead = int(np.prod(shapes[0][:ax]))
    tails = [int(np.prod(s[ax:])) for s in shapes]
    out = _empty((lead, sum(tails)), xs[0].data)
    col = 0
    for v, w in zip(xs, tails):
        t = E.contiguous(v).reshape(lead, w)
        K.copy2d(t, w, out, out.stride(0), lead, w, dst_off=col)
        col += w
    res = E.Var(out.reshape(out_shape))

    def bwd2(grads):
        g = grads[0].reshape(lead, -1)
        c = 0
        for v, w in zip(xs, tails):
            if v.requires_grad:
                gv = _empty((lead, w), g)
                K.copy2d(g, g.stride(0), gv, w, lead, w, src_off=c)
                E.add_grad(v, gv.reshape(v.data.shape))
            c += w

    E.record([res], xs, bwd2)
    return res


def slice_cols(x, col0, ncols, shape=None):
    """x[:, col0:col0+ncols] of the per-sample flattening."""
    b = x.data.shape[0]
    shape = shape or (b, ncols)
    if x.base is not None and x.ncols != -1:
        return _window(x.base, x.col0 + col0, ncols, shape)
    if x.data.dim() == 2 and x.base is None:
        return _window(x, col0, ncols, shape)
    src, ld = x.flat2d()
    out = _empty((b, ncols), x.data)
    K.copy2d(src, ld, out, ncols, b, ncols, src_off=col0)
    res = E.Var(out.reshape(shape))

    def bwd(grads):
        full = _empty((b, src.shape[1]), out)
        K.fill(full, 0.0)
        K.copy2d(grads[0].reshape(b, ncols), ncols, full, full.stride(0), b, ncols, dst_off=col0)
        E.add_grad(x, full.reshape(x.data.shape))

    E.record([res], [x], bwd)
    return res


def add_n(xs):
    """Keras Add on tensors with the same number of elements per sample ([B,1] / [B,1,1])."""
    xs = [v for v in xs]
    if len(xs) == 1:
        return xs[0]
    n = xs[0].data.numel()
    for v in xs:
        if v.data.numel() != n:
            raise ValueError("add_n: operands must have the same number of elements, got %s" %
                             [tuple(v.data.shape) for v in xs])
    ts = [E.contiguous(v).reshape(-1) for v in xs]
    out_t, i = None, 0
    while i < len(ts):                  # the kernel sums up to 8 operands per launch
        if out_t is None:
            chunk, i = ts[i:i + 8], i + 8
        else:
            chunk, i = [out_t] + ts[i:i + 7], i + 7
        out_t = K.add_n(chunk)
    best = max(xs, key=lambda v: v.data.dim())
    res = E.Var(out_t.reshape(best.data.shape) if best.data.dim() <= 2 else out_t.reshape(-1, 1))

    def bwd(grads):
        g = grads[0]
        for v in xs:
            if v.requires_grad:
                E.add_grad(v, g.reshape(v.data.shape))

    E.record([res], xs, bwd)
    return res


def add(x, y):
    """x + y for two tensors of the same shape (the Transformer's ``result += fw2``, layers/sequence.py:626)."""
    if tuple(x.shape) != tuple(y.shape):
        raise ValueError("add: shapes differ: %s vs %s" % (tuple(x.shape), tuple(y.shape)))
    res = E.Var(K.add_n([E.contiguous(x), E.contiguous(y)]))

    def bwd(grads):
        # x and y receive the same tensor: add_grad may adopt it as x.grad and later accumulate into it in place.
        # In the Transformer y (fw2) is produced after x and its backward runs next, before anything else adds
        # to x, so y has consumed the shared tensor by then.
        E.add_grad(x, grads[0])
        E.add_grad(y, grads[0])

    E.record([res], [x, y], bwd)
    return res


def rowsum(x):
    """sum over all non-batch axes -> [B,1]  (Linear mode 0/2, layers/utils.py:160-171)."""
    src, ld = x.flat2d()
    if src is None:
        t = E.contiguous(x)
        src = t.reshape(t.shape[0], -1)
        ld = src.stride(0)
    b, w = src.shape
    out = K.rowsum(src, b, w, ld)
    res = E.Var(out.reshape(b, 1))

    def bwd(grads):
        g = grads[0].reshape(b, 1)
        ones = _empty((1, w), g)
        K.fill(ones, 1.0)
        gx = K.gemm(g, ones, m=b, n=w, k=1)      # broadcast as an outer product
        E.add_grad(x, gx.reshape(x.data.shape))

    E.record([res], [x], bwd)
    return res


def zeros_like_batch(x, cols=1):
    b = x.data.shape[0]
    out = torch.empty((b, cols), dtype=torch.float32, device=x.data.device)
    K.fill(out, 0.0)
    return E.Var(out)


# ---- FM ------------------------------------------------------------------------------------------
def fm(x):
    """[B,F,E] -> [B,1]  (layers/interaction.py:597-602).  A ``ScaledFields`` input runs the field-weighted FM on its
    two factors (fm_weighted)."""
    if isinstance(x, ScaledFields):
        return fm_weighted(x.x, x.m)
    b, f, e = x.data.shape
    src, ld = x.flat2d()
    if src is None:
        t = E.contiguous(x)
        src, ld = t.reshape(b, f * e), f * e
    out = K.fm_fwd(src, f, e, ld)
    res = E.Var(out.reshape(b, 1))

    def bwd(grads):
        g = grads[0].reshape(b).contiguous()
        dx = _empty((b, f * e), g)
        L.check(L.lib().b2ctr_fm_bwd(K.ptr(src), ld, f, e, K.ptr(g), K.ptr(dx), f * e, 0, b, K.stream()),
                "fm_bwd")
        E.add_grad(x, dx.reshape(x.data.shape))

    E.record([res], [x], bwd)
    return res


# ---- field weights (IFM / DIFM) -------------------------------------------------------------------
class ScaledFields(E.Var):
    """The refine product x * expand_dims(m, -1) of IFM / DIFM (ifm.py:66-67, difm.py:74-75), kept as its two
    factors x [B,F,E] and m [B,F]: FM consumes them directly (fm_weighted), every other layer receives the
    materialised product (``product``, called by engine.Layer._invoke)."""
    __slots__ = ("x", "m", "_product")

    def __init__(self, x, m):
        E.Var.__init__(self, None, requires_grad=x.requires_grad or m.requires_grad, vshape=tuple(x.shape))
        self.x, self.m, self._product = x, m, None

    def product(self):
        if self._product is None:
            self._product = field_scale(self.x, self.m)
        return self._product


def scale_fields(x, m):
    """[B,F,E] x, [B,F] m -> x * m[:, :, None], deferred (``ScaledFields``): nothing is computed here."""
    if len(x.shape) != 3 or tuple(m.shape) != (x.shape[0], x.shape[1]):
        raise ValueError("scale_fields: x must be [B, F, E] and m [B, F], got %s and %s"
                         % (tuple(x.shape), tuple(m.shape)))
    return ScaledFields(x, m)


def _m2d(m, b, f):
    t = m.data
    if t.dim() == 2 and t.shape == (b, f) and t.stride(1) == 1:
        return t
    return E.contiguous(m).reshape(b, f)


def _grad_window(x, w):
    """(2-D view to write x's gradient into, accumulate) when x is a column window of a [B, ld] buffer: its slice of
    the buffer's gradient (added to when that exists; adopted as it, like engine.add_grad does, when x covers every
    used column), else (None, False)."""
    base = x.base
    if base is None or x.ncols == -1 or base.data is None or base.data.dim() != 2:
        return None, False
    if base.grad is not None:
        return base.grad[:, x.col0:x.col0 + w], True
    used = base.ncols if base.ncols > 0 else base.data.shape[1]
    if x.col0 == 0 and w >= used:
        base.grad = torch.empty_like(base.data)
        base.requires_grad = True
        return base.grad[:, :w], False
    return None, False


def fm_weighted(x, m):
    """[B,F,E] x, [B,F] m -> [B,1]: FM of m ⊙ x without writing m ⊙ x (b2ctr_fm_weighted_fwd).  x is read in place;
    the backward writes dx straight into the gather buffer's gradient when x is a window of it."""
    b, f, e = x.data.shape
    src, ld = _fields2d(x)
    md = _m2d(m, b, f)
    res = E.Var(K.fm_weighted_fwd(src, ld, md, f, e, b).reshape(b, 1))

    def bwd(grads):
        g = grads[0].reshape(b).contiguous()
        dxw, acc = _grad_window(x, f * e) if x.requires_grad else (None, False)
        dx, dm = K.fm_weighted_bwd(src, ld, md, f, e, g, b, dx=dxw, accumulate=acc, want_dx=x.requires_grad,
                                   want_dm=m.requires_grad)
        if x.requires_grad and dxw is None:
            E.add_grad(x, dx.reshape(x.data.shape))
        if dm is not None:
            E.add_grad(m, dm)

    E.record([res], [x, m], bwd)
    return res


def field_scale(x, m):
    """x * m over fields: x's per-sample values are F = m.shape[1] fields of dim values each ([B,F,E] for the FM
    input, [B,1,F] with dim 1 for the linear lookups of get_linear_logit).  Materialised, same shape as x."""
    b, f = m.shape
    src, ld = x.flat2d()
    if src is None:
        src = E.contiguous(x).reshape(b, -1)
        ld = src.stride(0)
    w = src.shape[1]
    if w % f:
        raise ValueError("field_scale: %d values per sample are not %d fields" % (w, f))
    dim = w // f
    md = _m2d(m, b, f)
    res = E.Var(K.field_scale_fwd(src, ld, md, f, dim, b).reshape(x.data.shape))

    def bwd(grads):
        g = grads[0].reshape(b, w)
        if not g.is_contiguous():
            g = g.contiguous()
        dxw, acc = _grad_window(x, w) if x.requires_grad else (None, False)
        dx, dm = K.field_scale_bwd(g, src, ld, md, f, dim, b, dx=dxw, accumulate=acc, want_dx=x.requires_grad,
                                   want_dm=m.requires_grad)
        if x.requires_grad and dxw is None:
            E.add_grad(x, dx.reshape(x.data.shape))
        if dm is not None:
            E.add_grad(m, dm)

    E.record([res], [x, m], bwd)
    return res


def _fields2d(x):
    """[B,F,E] -> (2-D [B, F*E] window, pitch): the fused gather's buffer is read in place."""
    b, f, e = x.data.shape
    src, ld = x.flat2d()
    if src is None:
        t = E.contiguous(x)
        src, ld = t.reshape(b, f * e), f * e
    return src, ld


def bi_interaction(x):
    """[B,F,E] -> [B,1,E]: 0.5 * ((sum_f x)^2 - sum_f x^2)  (BiInteractionPooling, layers/interaction.py:196-201)."""
    b, f, e = x.data.shape
    src, ld = _fields2d(x)
    out = K.bi_interaction_fwd(src, ld, f, e, b)
    res = E.Var(out.reshape(b, 1, e))

    def bwd(grads):
        g = grads[0].reshape(b, e)
        if not g.is_contiguous():
            g = g.contiguous()
        dx = K.bi_interaction_bwd(src, ld, f, e, g, b)
        E.add_grad(x, dx.reshape(x.data.shape))

    E.record([res], [x], bwd)
    return res


def afm(x, w, bias, h):
    """[B,F,E] -> [B,E]: attention-weighted sum of the pairwise products v_i * v_j (AFMLayer up to its dropout,
    layers/interaction.py:126-141).  The [B, P, E] products and the [B, P, A] attention hidden layer are generated
    on chip in the forward and again in the backward; only a [B, 2] softmax state is kept."""
    b, f, e = x.data.shape
    src, ld = _fields2d(x)
    wd, bd, hd = _wdata(w), _wdata(bias), _wdata(h)
    att, state = K.afm_fwd(src, ld, f, e, wd, bd, hd.reshape(-1), b)
    res = E.Var(att)

    def bwd(grads):
        g = grads[0].reshape(b, e)
        if not g.is_contiguous():
            g = g.contiguous()
        dx, dw, db, dh = K.afm_bwd(g, src, ld, f, e, wd, bd, hd.reshape(-1), state, att, b)
        E.add_grad(x, dx.reshape(x.data.shape))
        if w.requires_grad:
            E.add_grad(w, dw)
        if bias.requires_grad:
            E.add_grad(bias, db.reshape(bd.shape))
        if h.requires_grad:
            E.add_grad(h, dh.reshape(hd.shape))

    E.record([res], [x, w, bias, h], bwd)
    return res


def senet(x, w1, w2):
    """[B,F,E] -> V [B,F,E]: x reweighted by relu(relu(mean_e(x) W1) W2) (SENETLayer, layers/interaction.py:1119-1124).
    x is read in place; only V and the [B, R + F] excitation (A1, A2) are written."""
    b, f, e = x.data.shape
    src, ld = _fields2d(x)
    w1d, w2d = _wdata(w1), _wdata(w2)
    v, saved = K.senet_fwd(src, ld, f, e, w1d, w2d, b)
    res = E.Var(v)                       # [B, F*E]: the layer hands out per-field windows of it

    def bwd(grads):
        g = grads[0]
        if not g.is_contiguous():
            g = g.contiguous()
        dx, dw1, dw2 = K.senet_bwd(g.reshape(b, f * e), src, ld, f, e, w1d, w2d, saved, b)
        E.add_grad(x, dx.reshape(x.data.shape))
        if w1.requires_grad:
            E.add_grad(w1, dw1)
        if w2.requires_grad:
            E.add_grad(w2, dw2)

    E.record([res], [x, w1, w2], bwd)
    return res


def bilinear_interaction(x, weights, stack, btype, out=None):
    """[B,F,E] -> [B,P,E]: (v_i W_k) * v_j for the pairs i < j (BilinearInteraction, layers/interaction.py:1196-1208).
    ``stack`` [nW,E,E] holds the data of ``weights`` (each weight's data is a view of it); the gradient comes back
    as one stacked buffer handed to each weight as a view.  ``out``: a strided [B,P,E] view of a wider buffer to
    write the pairs into (the DNN input, see inputs.DnnInputPlacement); default a new [B,P,E] tensor."""
    b, f, e = x.data.shape
    P = f * (f - 1) // 2
    src, ld = _fields2d(x)
    if out is None:
        out = K.bilinear_fwd(src, ld, f, e, btype, stack, b).reshape(b, P, e)
    else:
        K.bilinear_fwd(src, ld, f, e, btype, stack, b, out=out, col0=0, pitch=out.stride(1))
    res = E.Var(out)

    def bwd(grads):
        g = grads[0].reshape(b, P, e)
        if g.stride(2) != 1 or g.stride(1) < e:
            g = g.contiguous()
        want_dw = any(w.requires_grad for w in weights)
        dx, dw = K.bilinear_bwd(g, g.stride(0), 0, g.stride(1), src, ld, f, e, btype, stack, b,
                                want_dx=x.requires_grad, want_dw=want_dw)
        if dx is not None:
            E.add_grad(x, dx.reshape(x.data.shape))
        for k, w in enumerate(weights):
            if w.requires_grad:
                E.add_grad(w, dw[k])

    E.record([res], [x] + list(weights), bwd)
    return res


def fwfm(x, r):
    """[B,F,E] -> [B,1]: sum_{i<j} r[i,j] <x_i, x_j> over the upper triangle of r [F,F] (FwFMLayer,
    layers/interaction.py:1403-1411).  x is read in place; the gradient of r is 0 on and below the diagonal."""
    b, f, e = x.data.shape
    src, ld = _fields2d(x)
    rd = _wdata(r)
    res = E.Var(K.fwfm_fwd(src, ld, f, e, rd, b))

    def bwd(grads):
        if not (x.requires_grad or r.requires_grad):
            return
        g = grads[0].reshape(b, 1)
        if not g.is_contiguous():
            g = g.contiguous()
        dx, dr = K.fwfm_bwd(g, g.stride(0), src, ld, f, e, rd, b, want_dx=x.requires_grad, want_dr=r.requires_grad)
        if dx is not None:
            E.add_grad(x, dx.reshape(x.data.shape))
        if dr is not None:
            E.add_grad(r, dr)

    E.record([res], [x, r], bwd)
    return res


def fefm(x, weights, stack, out=None):
    """[B,F,E] -> [B,P]: x_i (W_p + W_p^T) x_j^T for the pairs p = (i < j) (FEFMLayer, layers/interaction.py:1481-1491).
    ``stack`` [P,E,E] holds the data of ``weights`` (each weight's data is a view of it); the symmetric S_p are
    built once per call and the gradient comes back as one stacked buffer handed to each weight as a view.
    x is read in place; no per-pair [B,E] product is written.

    ``out``: a [B,P] column window (``_window``) of a wider buffer Var to write the scores into (DeepFEFM's DNN
    input behind the gather buffer's dense columns, inputs.EmbeddingPlanner._fefm_scores); it is returned.  Every
    consumer's gradient then lands in that buffer's gradient, so the backward is keyed on the buffer: it reads the
    score columns of its gradient in place and leaves the gradient to the buffer's own backward (the gather's
    scatter), which runs after it.  Default: a new [B,P] tensor."""
    b, f, e = x.data.shape
    src, ld = _fields2d(x)
    S = K.fefm_sym(stack)
    if out is None:
        res = E.Var(K.fefm_fwd(src, ld, f, e, S, b))
        key, gcol0 = res, 0
    else:
        key, gcol0 = out.base, out.col0
        K.fefm_fwd(src, ld, f, e, S, b, out=key.data, col0=gcol0)
        res = out

    def bwd(grads):
        g = grads[0]
        if g.dim() != 2 or g.stride(1) != 1 or g.stride(0) < g.shape[1]:
            g = g.contiguous().reshape(b, -1)
        want_dw = any(w.requires_grad for w in weights)
        if not (x.requires_grad or want_dw):
            return
        dx, dw = K.fefm_bwd(g, g.stride(0), gcol0, src, ld, f, e, S, b, want_dx=x.requires_grad, want_dw=want_dw)
        if dx is not None:
            E.add_grad(x, dx.reshape(x.data.shape))
        for k, w in enumerate(weights):
            if w.requires_grad:
                E.add_grad(w, dw[k])

    if E.record([key], [x] + list(weights), bwd, keep_grads=out is not None):
        res.requires_grad = True
    return res


def _pair_grad(grads, b):
    g = grads[0]
    if g.dim() != 2 or g.stride(1) != 1 or g.stride(0) < g.shape[1]:
        g = g.contiguous().reshape(b, -1)
    return g


def pnn_inner(x, mode, kernel=None, out=None):
    """[B,F,E] -> PNN's pairwise products for the pairs p = (i < j) (b2ctr_pnn_inner_fwd): mode 'inner'
    <x_i, x_j> as [B,P,1] (InnerProductLayer, layers/interaction.py:669-678), 'elementwise' x_i * x_j as [B,P,E]
    (reduce_sum=False), 'vec' / 'num' the kernel-weighted inner products as [B,P] (OutterProductLayer,
    :912-919, with ``kernel`` [P,E] / [P,1]).  x is read in place.

    ``out``: a [B,P] column window (``_window``) of a wider buffer Var to write the scores into (PNN's DNN input,
    inputs.EmbeddingPlanner._pnn_products); the result is then a window of that buffer.  Every consumer's gradient
    lands in that buffer's gradient, so the backward is keyed on the buffer: it reads the score columns of its
    gradient in place and leaves the gradient to the buffer's own backward (the gather's scatter), as ops.fefm."""
    b, f, e = x.data.shape
    P = f * (f - 1) // 2
    src, ld = _fields2d(x)
    kd = _wdata(kernel) if kernel is not None else None
    shape = {"inner": (b, P, 1), "elementwise": (b, P, e)}.get(mode, (b, P))
    if out is None:
        res = E.Var(K.pnn_inner_fwd(src, ld, f, e, mode, kd, b).reshape(shape))
        key, gcol0 = res, 0
    else:
        key, gcol0 = out.base, out.col0
        K.pnn_inner_fwd(src, ld, f, e, mode, kd, b, out=key.data, col0=gcol0)
        res = _window(key, gcol0, P, shape)
    wts = [kernel] if kernel is not None else []

    def bwd(grads):
        want_dk = kernel is not None and kernel.requires_grad
        if not (x.requires_grad or want_dk):
            return
        g = _pair_grad(grads, b)
        dx, dk = K.pnn_inner_bwd(g, g.stride(0), gcol0, src, ld, f, e, mode, kd, b, want_dx=x.requires_grad,
                                 want_dk=want_dk)
        if dx is not None:
            E.add_grad(x, dx.reshape(x.data.shape))
        if dk is not None:
            E.add_grad(kernel, dk)

    if E.record([key], [x] + wts, bwd, keep_grads=out is not None):
        res.requires_grad = True
    return res


def pnn_outer(x, kernel, out=None):
    """[B,F,E] -> [B,P]: sum_{k,l} x_j[k] K[k,p,l] x_i[l] for the pairs p = (i < j) (OutterProductLayer
    kernel_type='mat', layers/interaction.py:881-911), with the kernel [E,P,E] read in place by the FEFM tiles
    (b2ctr_pnn_outer_fwd): no per-pair [B,E] product is written.  ``out`` as in pnn_inner."""
    b, f, e = x.data.shape
    src, ld = _fields2d(x)
    kd = _wdata(kernel)
    if out is None:
        res = E.Var(K.pnn_outer_fwd(src, ld, f, e, kd, b))
        key, gcol0 = res, 0
    else:
        key, gcol0 = out.base, out.col0
        K.pnn_outer_fwd(src, ld, f, e, kd, b, out=key.data, col0=gcol0)
        res = out

    def bwd(grads):
        if not (x.requires_grad or kernel.requires_grad):
            return
        g = _pair_grad(grads, b)
        dx, dk = K.pnn_outer_bwd(g, g.stride(0), gcol0, src, ld, f, e, kd, b, want_dx=x.requires_grad,
                                 want_dk=kernel.requires_grad)
        if dx is not None:
            E.add_grad(x, dx.reshape(x.data.shape))
        if dk is not None:
            E.add_grad(kernel, dk)

    if E.record([key], [x, kernel], bwd, keep_grads=out is not None):
        res.requires_grad = True
    return res


def add_bias(x, b, scale=1.0, per_sample=False):
    """x + scale * b over the last axis for a per-column (or scalar, when the last axis is 1) bias:
    Linear(use_bias=True) without a dense part, layers/utils.py:172-173.  ``per_sample``: b spans every non-batch
    axis (PositionEncoding's x + sqrt(E) P[t] over the [B, T*E] view, layers/sequence.py:683-689).  Forward = copy
    + rank-1 update ones[B,1] @ b[1,n] through the skinny GEMM kernel; backward = pass-through and a column sum."""
    xt = E.contiguous(x)
    x2 = xt.reshape(xt.shape[0], -1) if per_sample else xt.reshape(-1, xt.shape[-1])
    m, n = x2.shape
    bd = b.materialize() if isinstance(b, E.Weight) else b.data
    if bd.numel() != n:
        raise ValueError("add_bias: bias has %d elements, last axis has %d" % (bd.numel(), n))
    y = K.add_n([x2])                                     # copy
    ones = K.fill(torch.empty((m, 1), dtype=torch.float32, device=y.device), 1.0)
    K.gemm(ones, bd.reshape(1, n), c=y, accumulate=True, alpha=scale, m=m, n=n, k=1)
    out = E.Var(y.reshape(x.data.shape), mask=x.mask if per_sample else None)

    def bwd(grads):
        dy = grads[0]
        if x.requires_grad:
            E.add_grad(x, dy)
        if b.requires_grad:
            dy2 = dy.reshape(m, n)
            if not dy2.is_contiguous():
                dy2 = dy2.contiguous()
            _, db = K.bias_act_bwd(dy2, None, L.ACT_NONE, want_dz=False, want_dbias=True)
            if scale != 1.0:
                db = K.add_n([db], scales=[scale], out=db)
            E.add_grad(b, db.reshape(bd.shape))

    E.record([out], [x, b], bwd)
    return out


# ==================================================================================================
# interaction operators
# ==================================================================================================
def _wdata(w):
    return w.materialize() if isinstance(w, E.Weight) else w.data


def _rows2d(x):
    """[B, d] window -> (tensor2d, ld)."""
    t, ld = x.flat2d()
    if t is None:
        t = E.contiguous(x).reshape(x.shape[0], -1)
        ld = t.stride(0)
    return t, ld


def cross_vector(x0, xl, w, bias):
    """x_{l+1} = x_0 * (x_l . w) + b + x_l   (layers/interaction.py:413-416)."""
    t0, ld0 = _rows2d(x0)
    tl, ldl = _rows2d(xl)
    b, d = t0.shape
    wd, bd = _wdata(w), _wdata(bias)
    out, s = K.cross_vector_fwd(t0, ld0, tl, ldl, wd, bd, b, d)
    res = E.Var(out)

    def bwd(grads):
        g = grads[0]
        if not g.is_contiguous():
            g = g.contiguous()
        dx0, dxl, ds = K.cross_vector_bwd(t0, ld0, wd, g, s, b, d)
        E.add_grad(x0, dx0)
        E.add_grad(xl, dxl)
        if w.requires_grad:
            dw = K.gemm(tl, ds.reshape(b, 1), trans_a=True, split_k=_split_k(d, 1, b), m=d, n=1, k=b)
            E.add_grad(w, dw.reshape(w.shape))
        if bias.requires_grad:
            _, db = K.bias_act_bwd(g, None, L.ACT_NONE, want_dz=False, want_dbias=True)
            E.add_grad(bias, db.reshape(bias.shape))

    E.record([res], [x0, xl, w, bias], bwd)
    return res


def cross_matrix(x0, xl, w, bias):
    """x_{l+1} = x_0 * (W x_l + b) + x_l   (layers/interaction.py:417-420)."""
    t0, ld0 = _rows2d(x0)
    tl, ldl = _rows2d(xl)
    b, d = t0.shape
    wd, bd = _wdata(w), _wdata(bias).reshape(-1)
    c0 = E.contiguous(x0).reshape(b, d) if ld0 != d else t0
    cl = E.contiguous(xl).reshape(b, d) if ldl != d else tl
    u = K.gemm(cl, wd, bias=bd, trans_b=True, precision=GEMM_PRECISION, m=b, n=d, k=d)     # W x_l + b
    out = K.ewise(1, c0, u, cl)                                                           # x0*u + xl
    res = E.Var(out)

    def bwd(grads):
        g = grads[0]
        if not g.is_contiguous():
            g = g.contiguous()
        du = K.ewise(0, g, c0)
        E.add_grad(x0, K.ewise(0, g, u))
        dxl = K.gemm(du, wd, precision=GEMM_PRECISION, m=b, n=d, k=d)                     # du @ W
        K.axpy(g, dxl, 1.0)
        E.add_grad(xl, dxl)
        if w.requires_grad:
            dw = K.gemm(du, cl, trans_a=True, precision=GEMM_PRECISION, split_k=_split_k(d, d, b), m=d, n=d, k=b)
            E.add_grad(w, dw)
        if bias.requires_grad:
            _, db = K.bias_act_bwd(du, None, L.ACT_NONE, want_dz=False, want_dbias=True)
            E.add_grad(bias, db.reshape(bias.shape))

    E.record([res], [x0, xl, w, bias], bwd)
    return res


def _row_fields(d):
    """(fields, dim) splitting a row of d values for b2ctr_regulate when no gate gives it fields: the largest dim
    within the kernel's limits, a multiple of 4 where one divides d (its 16-byte path).  Without gates the split
    does not change the result."""
    fits = [e for e in range(min(d, K.REGULATE_MAX_DIM), 0, -1) if d % e == 0 and d // e <= K.REGULATE_MAX_FIELDS]
    if not fits:
        raise ValueError("a bridge over %d columns exceeds the regulate kernel's %d x %d limit"
                         % (d, K.REGULATE_MAX_FIELDS, K.REGULATE_MAX_DIM))
    e = next((e for e in fits if e % 4 == 0), fits[0])
    return d // e, e


def regulate(mode, x, h=None, ax=None, ah=None, gates=(), want_u=True):
    """EDCN's BridgeModule and RegulationModules in one launch (b2ctr_regulate_fwd): v = x ('copy'), x + h ('add'),
    x * h ('hadamard') or ax * x + ah * h ('attention') over [B, d] rows read in place, then u = v (when ``want_u``)
    and y_k = v * softmax_f(g_k * inv_tau_k) per field for each gate (g_k the RegulationModule weight [1, F, 1],
    inv_tau_k its stored 1 / tau).  Returns (u or None, [y_k]), each [B, d].  The backward recomputes v, writes dx
    straight into the gather buffer's gradient when x is a window of it, and reduces the gate gradients in a fixed
    order (b2ctr_regulate_bwd)."""
    b = x.shape[0]
    ops_ = [x, h, ax, ah]
    t2 = [_rows2d(v)[0] if v is not None else None for v in ops_]
    d = t2[0].shape[1]
    for v in t2[1:]:
        if v is not None and v.shape[1] != d:
            raise ValueError("regulate: operands of %d and %d columns" % (d, v.shape[1]))
    if gates:
        f = int(gates[0][0].shape[1])
        if d % f:
            raise ValueError("regulate: %d columns are not %d fields" % (d, f))
        e = d // f
    else:
        f, e = _row_fields(d)
    if not (1 <= f <= K.REGULATE_MAX_FIELDS and 1 <= e <= K.REGULATE_MAX_DIM):
        raise ValueError("RegulationModule supports 1 to %d fields and embedding_size 1 to %d (got %d fields, "
                         "embedding_size %d)" % (K.REGULATE_MAX_FIELDS, K.REGULATE_MAX_DIM, f, e))
    kg = [(_wdata(g).reshape(-1), it) for g, it in gates]
    outs = [_empty((b, d), t2[0]) for _ in range(int(bool(want_u)) + len(gates))]
    u = outs[0] if want_u else None
    ys = outs[1:] if want_u else outs
    K.regulate_fwd(mode, f, e, b, t2[0], t2[1], t2[2], t2[3], kg, u=(u, 0) if u is not None else None,
                   y0=(ys[0], 0) if len(ys) > 0 else None, y1=(ys[1], 0) if len(ys) > 1 else None)
    res = [E.Var(o) for o in outs]

    def bwd(grads):
        gs = [_pair_grad([g], b) if g is not None else None for g in grads]
        gu = gs[0] if want_u else None
        gy = (gs[1:] if want_u else gs) + [None, None]
        want_dg = [gy[k] is not None and gates[k][0].requires_grad for k in range(len(gates))] + [False, False]
        want = [v is not None and v.requires_grad for v in ops_]
        if not (any(want) or any(want_dg)):
            return
        dxw, acc = _grad_window(x, d) if x.requires_grad else (None, False)
        win = lambda g: (g, 0) if g is not None else None   # noqa: E731
        dx, dh, dax, dah, dg0, dg1 = K.regulate_bwd(
            mode, f, e, b, t2[0], t2[1], t2[2], t2[3], kg, du=win(gu), dy0=win(gy[0]), dy1=win(gy[1]),
            want_dx=want[0], dx=dxw, dx_accumulate=acc, want_dh=want[1], want_dax=want[2], want_dah=want[3],
            want_dg=want_dg[:2])
        if x.requires_grad and dxw is None:
            E.add_grad(x, dx.reshape(x.data.shape))
        for v, g in ((h, dh), (ax, dax), (ah, dah)):
            if g is not None:
                E.add_grad(v, g.reshape(v.data.shape))
        for (w, _), g in zip(gates, (dg0, dg1)):
            if g is not None:
                E.add_grad(w, g.reshape(w.shape))

    E.record(res, [v for v in ops_ if v is not None] + [g for g, _ in gates], bwd)
    return (res[0] if want_u else None), (res[1:] if want_u else res)



def conv_stack(x, stages, rows, dim, channels, out_shape):
    """CCPM's Conv2D / KMaxPooling stages (deepctr/models/ccpm.py:58-70) on x viewed as [n, rows, dim, channels]
    (n = the elements of x over rows * dim * channels), one b2ctr_conv_stack launch for all of them: every
    (n, dim) column runs the whole stack on chip and only the last map is written, as a new [n, k * dim * C] tensor
    reshaped to ``out_shape``.  ``stages``: ("conv", width, filters, activation, kernel Weight, bias Weight or None)
    or ("kmax", k).  x is read in place when it is a window of a wider buffer (the gather buffer); the backward
    recomputes the stack, adds dx to that buffer's gradient and sums the weight gradients in a fixed order."""
    w_in = rows * dim * channels
    src, _ = _rows2d(x) if x.data.dim() >= 2 else (None, 0)
    if src is None or src.shape[1] != w_in:
        src = E.contiguous(x).reshape(-1, w_in)
    n = src.shape[0]
    kst = [st if st[0] != "conv" else st[:4] + (_wdata(st[4]), _wdata(st[5]) if st[5] is not None else None)
           for st in stages]
    k_out, c_out = K.conv_stack_check(rows, channels, stages)
    w_out = k_out * dim * c_out
    y = _empty((n, w_out), src)
    K.conv_stack_fwd(kst, src, rows, dim, channels, n, y)
    res = E.Var(y.reshape(out_shape))
    weights = [w for st in stages if st[0] == "conv" for w in st[4:] if w is not None]

    def bwd(grads):
        want_dw = [st[0] == "conv" and (st[4].requires_grad or (st[5] is not None and st[5].requires_grad))
                   for st in stages]
        if not (x.requires_grad or any(want_dw)):
            return
        g = grads[0].reshape(n, w_out)
        if not g.is_contiguous():
            g = g.contiguous()
        dxw, acc = (None, False)
        if x.requires_grad:
            dxw, acc = _grad_window(x, w_in) if src.shape[0] == x.data.shape[0] else (None, False)
        dx = dxw if dxw is not None else (_empty((n, w_in), g) if x.requires_grad else None)
        dws = K.conv_stack_bwd(kst, src, rows, dim, channels, n, g, dx=dx, dx_accumulate=acc, want_dw=want_dw)
        if x.requires_grad and dxw is None:
            E.add_grad(x, dx.reshape(x.data.shape))
        for st, d in zip(stages, dws):
            if d is not None:
                E.add_grad(st[4], d[0])
                if d[1] is not None:
                    E.add_grad(st[5], d[1])

    E.record([res], [x] + weights, bwd)
    return res

def field_wise_bi(groups, kernel_mf, kernel_fm, bias_mf=None, bias_fm=None):
    """FLEN's FieldWiseBiInteraction (deepctr/layers/interaction.py:1283-1337) in one b2ctr_field_wise_bi launch.
    ``groups``: G lists of [B, n, E] tensors, the members of each group (a group is the field axis concatenation of
    its list).  When every member is a column window of one buffer (the gather buffer) the fields are read there in
    place, whether or not a group's members are adjacent; otherwise the members are first copied into one
    [B, F, E] buffer.  Returns h [B, E]; only h is written.  The backward recomputes the group sums, adds dx into
    that buffer's gradient (or writes it into the copy's) and sums the weight gradients in a fixed order."""
    members = [m for g in groups for m in g]
    b, e = members[0].data.shape[0], members[0].data.shape[-1]
    G = len(groups)
    nf = [int(np.prod(m.data.shape[1:])) // e for m in members]
    K.field_wise_bi_check(sum(nf), G, e)
    gid = [k for k, g in enumerate(groups) for _ in g]
    base = members[0].base
    in_place = (base is not None and base.data is not None and base.data.dim() == 2
                and all(m.base is base and m.ncols != -1 and m.data is not None for m in members))
    if in_place:
        x, src = None, base.data
        cols = [m.col0 + i * e for m, n in zip(members, nf) for i in range(n)]
    else:
        x = concat(members, 1)
        src = E.contiguous(x).reshape(b, -1)
        cols = [i * e for i in range(sum(nf))]
    fgroup = [k for k, n in zip(gid, nf) for _ in range(n)]
    w = [_wdata(v) if v is not None else None for v in (kernel_mf, kernel_fm, bias_mf, bias_fm)]
    h = _empty((b, e), src)
    K.field_wise_bi_fwd(src, cols, fgroup, G, e, b, w[0], w[1], w[2], w[3], h)
    res = E.Var(h)
    weights = [v for v in (kernel_mf, kernel_fm, bias_mf, bias_fm) if v is not None]
    xs = members if in_place else [x]

    def bwd(grads):
        want_dx = any(v.requires_grad for v in xs)
        want_dk = (kernel_mf.requires_grad, kernel_fm.requires_grad)
        want_db = tuple(v is not None and v.requires_grad for v in (bias_mf, bias_fm))
        if not (want_dx or any(want_dk) or any(want_db)):
            return
        g = grads[0].reshape(b, e)
        if not g.is_contiguous():
            g = g.contiguous()
        dx, acc = None, False
        if want_dx and in_place:
            if base.grad is None:
                base.grad = torch.empty_like(base.data)
                K.fill(base.grad, 0.0)
                base.requires_grad = True
            dx, acc = base.grad, True
        elif want_dx:
            dx = _empty((b, src.shape[1]), g)
        dkm, dkf, dbm, dbf = K.field_wise_bi_bwd(src, cols, fgroup, G, e, b, w[0], w[1], w[2], w[3], g, dx=dx,
                                                 dx_accumulate=acc, want_dkernel=want_dk, want_dbias=want_db)
        if want_dx and not in_place:
            E.add_grad(x, dx.reshape(x.data.shape))
        for v, d in ((kernel_mf, dkm), (kernel_fm, dkf), (bias_mf, dbm), (bias_fm, dbf)):
            if d is not None:
                E.add_grad(v, d)

    E.record([res], xs + weights, bwd)
    return res


CIN_CHUNK_BYTES = 24 << 20      # outer-product chunk kept well inside the 50 MB L2


CIN_FOLD = True               # fused CIN: fold dZ = dY W^T onto the factors inside the GEMM epilogue (b2ctr_cin_fold)
CIN_DZ_CHUNK_BYTES = 512 << 20


def cin_fusable(x, layer_size, split_half):
    """The outer product can be generated inside the wgmma GEMM producer (b2ctr_cin_gemm)."""
    B, m, D = x.shape
    hid = [n // 2 if split_half else n for n in layer_size[:-1]]
    return (GEMM_PRECISION == L.GEMM_BF16X3 and B * D >= 256 and D in (4, 8, 16, 32, 64, 128)
            and min(layer_size) >= 8 and all(n % 4 == 0 for n in layer_size) and all(h % 4 == 0 for h in hid))


def cin(x, filters, biases, layer_size, activation, split_half):
    with K.profile_tag("cin"):
        if cin_fusable(x, layer_size, split_half):
            return _cin_fused(x, filters, biases, layer_size, activation, split_half)
        return _cin(x, filters, biases, layer_size, activation, split_half)


def _cin_pad(h):
    return 32 if h <= 32 else (h + 63) // 64 * 64


def _cin_fused(x, filters, biases, layer_size, activation, split_half):
    """CIN (layers/interaction.py:277-325) with the outer product Z[(b,d), (i,j)] = X0(b,i,d) X_k(b,j,d) GENERATED
    by the producer warps of the tensor-core GEMM instead of being written anywhere: forward Y = act(Z W + b) and
    the filter gradient dW = Z^T dY both read only the two factors (T0 = X0 transposed to [(b,d), m], X_k as the
    previous layer's [(b,d), N] activations).  Only dZ = dY W^T of the backward pass exists in memory, in row chunks."""
    B, m, D = x.shape
    x2, ldx = x.flat2d()
    if x2 is None:
        x2 = E.contiguous(x).reshape(B, m * D)
        ldx = m * D
    act = L.ACT_BY_NAME[activation]
    nl = len(layer_size)
    hs = [m] + [size // 2 if split_half else size for size in layer_size]
    direct = [((size // 2, size // 2) if (split_half and i != nl - 1) else (0, size)) for i, size in enumerate(layer_size)]
    out_cols = sum(nc for _, nc in direct)
    out = _empty((B, out_cols), x2)
    rows = B * D
    v0 = (ldx, D, 1)
    ld0 = 32 if m <= 32 else (m + 63) // 64 * 64
    t0 = K.cin_t0(x2, v0, B, m, D, ld0)                       # [rows, ld0]
    tv0 = (D * ld0, 1, ld0)                                   # T0 seen as X0(b,i,d)
    ws2d = [_wdata(f).reshape(-1, f.shape[-1]) for f in filters]
    bs = [_wdata(bv) for bv in biases]
    hps = [_cin_pad(hs[i]) for i in range(nl)]
    wplanes, ys = [], []
    oc = 0
    for i, size in enumerate(layer_size):
        h, hp = hs[i], hps[i]
        xk, ldk = (t0, ld0) if i == 0 else (ys[-1], layer_size[i - 1])
        wp = K.cin_filter_planes(ws2d[i], m, h, hp)
        y = K.cin_gemm(0, t0, xk, ldk, rows, m, h, hp, size, wp, bias=bs[i], act=act)
        K.cin_sum_d(y, size, direct[i][0], direct[i][1], D, out, out_cols, oc, 0, B)
        oc += direct[i][1]
        wplanes.append(wp)
        ys.append(y)
    res = E.Var(out)

    def bwd(grads):
        g = grads[0]
        if not g.is_contiguous():
            g = g.contiguous()
        gx = (m * D, D, 1)
        fold = CIN_FOLD and all(hp in (32, 64, 128) for hp in hps)
        dx = _empty((B, m * D), x2)
        if fold:
            dt0 = _empty((rows, ld0), x2)          # gradient of the factor table, all layers accumulate into it
            K.fill(dt0, 0.0)
        else:
            K.fill(dx, 0.0)
        dh = None
        col = out_cols
        for i in range(nl - 1, -1, -1):
            size, h, hp = layer_size[i], hs[i], hps[i]
            kq = m * hp
            col -= direct[i][1]
            dy = _empty((rows, size), x2)
            K.cin_expand_grad(g, out_cols, col, direct[i][0], direct[i][1], dh, hs[i + 1] if dh is not None else 0,
                              hs[i + 1] if dh is not None else 0, dy, size, D, 0, B)
            if act != L.ACT_NONE and K.planes_fusable(rows, size):
                dz_, db, dzp = K.bias_act_bwd(dy, ys[i], act, want_dz=True, want_dbias=True, want_planes=True)
            else:
                dz_, db = K.bias_act_bwd(dy, ys[i], act, want_dz=act != L.ACT_NONE, want_dbias=True)
                if dz_ is None:
                    dz_ = dy
                dzp = K.split_planes(dz_)
            E.add_grad(biases[i], db)
            xk, ldk = (t0, ld0) if i == 0 else (ys[i - 1], layer_size[i - 1])
            xkv = tv0 if i == 0 else (D * layer_size[i - 1], 1, layer_size[i - 1])
            if filters[i].requires_grad:
                dwp = K.cin_gemm(1, t0, xk, ldk, rows, m, h, hp, size, dzp, split_k=_split_k(kq, size, rows))
                E.add_grad(filters[i], K.cin_unpad_rows(dwp, m, h, hp).reshape(filters[i].shape))
            dhid = None
            if fold:
                # dZ = dY W'^T exists only as accumulator tiles: the GEMM epilogue folds it onto T0 and X_k
                if i > 0:
                    dhid = _empty((rows, h), x2)
                    K.fill(dhid, 0.0)
                K.cin_fold(t0, xk, ldk, rows, m, h, hp, size, wplanes[i], dzp, dt0, dt0 if i == 0 else dhid,
                           ld0 if i == 0 else h)
            else:
                # dZ in row chunks, folded back onto the two factors by a second kernel
                dhid = _empty((rows, h), x2) if i > 0 else None
                chunk = max(256, min(rows, CIN_DZ_CHUNK_BYTES // (4 * kq)) // 256 * 256)
                dzf = _empty((min(chunk, rows), kq), x2)
                for r0 in range(0, rows, chunk):
                    nr = min(chunk, rows - r0)
                    K.gemm(dz_[r0:r0 + nr], dz_, c=dzf[:nr], trans_b=True, precision=L.GEMM_BF16X3, m=nr, n=kq, k=size,
                           b_planes=wplanes[i])
                    b0, nbk = r0 // D, nr // D
                    if i == 0:
                        K.cin_outer_bwd(dzf, t0, tv0, t0, tv0, dx, gx, True, dx, gx, True, b0, nbk, m, h, D, hp)
                    else:
                        K.cin_outer_bwd(dzf, t0, tv0, ys[i - 1], xkv, dx, gx, True, dhid, (D * h, 1, h), False, b0, nbk,
                                        m, h, D, hp)
            dh = dhid
        if fold:
            K.cin_t0_bwd(dt0, ld0, dx, gx, False, B, m, D)
        E.add_grad(x, dx.reshape(x.shape))

    E.record([res], [x] + list(filters) + list(biases), bwd)
    return res


def _cin(x, filters, biases, layer_size, activation, split_half):
    """Compressed Interaction Network (layers/interaction.py:277-325).  Per batch chunk the outer
    product Z[(b,d), i*H+j] lives in an L2-sized scratch buffer and is contracted with the filter by
    b2ctr_gemm; layer outputs are kept as [B, D, N] so the next layer reads them through strides."""
    B, m, D = x.shape
    x2, ldx = x.flat2d()
    if x2 is None:
        x2 = E.contiguous(x).reshape(B, m * D)
        ldx = m * D
    act = L.ACT_BY_NAME[activation]
    nl = len(layer_size)
    hs = [m]
    for i, size in enumerate(layer_size):
        hs.append(size // 2 if split_half else size)
    direct = []            # (col0, ncols) of each layer's direct maps
    for i, size in enumerate(layer_size):
        if split_half and i != nl - 1:
            direct.append((size // 2, size // 2))
        else:
            direct.append((0, size))
    out_cols = sum(nc for _, nc in direct)
    out = _empty((B, out_cols), x2)
    v0 = (ldx, D, 1)
    ys = []                # per layer activations [B*D, N]
    kmax = max(m * hs[i] for i in range(nl))
    chunk = max(1, min(B, CIN_CHUNK_BYTES // (4 * D * kmax)))
    z = _empty((chunk * D, kmax), x2)
    ws = [_wdata(f).reshape(-1, f.shape[-1]) for f in filters]
    bs = [_wdata(bv) for bv in biases]
    oc = 0
    for i, size in enumerate(layer_size):
        h = hs[i]
        kdim = m * h
        y = _empty((B * D, size), x2)
        src, vk = (x2, v0) if i == 0 else (ys[-1], (D * layer_size[i - 1], 1, layer_size[i - 1]))
        for b0 in range(0, B, chunk):
            nb = min(chunk, B - b0)
            zc = z.reshape(-1)[:nb * D * kdim].reshape(nb * D, kdim)
            K.cin_outer_fwd(x2, v0, src, vk, zc, b0, nb, m, h, D)
            K.gemm(zc, ws[i], c=y[b0 * D:(b0 + nb) * D], bias=bs[i], act=act, precision=GEMM_PRECISION,
                   m=nb * D, n=size, k=kdim)
        K.cin_sum_d(y, size, direct[i][0], direct[i][1], D, out, out_cols, oc, 0, B)
        oc += direct[i][1]
        ys.append(y)
    res = E.Var(out)

    def bwd(grads):
        with K.profile_tag("cin"):
            _bwd(grads)

    def _bwd(grads):
        g = grads[0]
        if not g.is_contiguous():
            g = g.contiguous()
        dx = _empty((B, m * D), x2)
        K.fill(dx, 0.0)
        gx = (m * D, D, 1)
        dh = None                                    # gradient wrt the hidden maps feeding layer i+1
        col = out_cols
        for i in range(nl - 1, -1, -1):
            size, h = layer_size[i], hs[i]
            kdim = m * h
            col -= direct[i][1]
            dy = _empty((B * D, size), x2)
            K.cin_expand_grad(g, out_cols, col, direct[i][0], direct[i][1], dh, hs[i + 1] if dh is not None else 0,
                              hs[i + 1] if dh is not None else 0, dy, size, D, 0, B)
            dz_, db = K.bias_act_bwd(dy, ys[i], act, want_dz=act != L.ACT_NONE, want_dbias=True)
            if dz_ is None:
                dz_ = dy
            E.add_grad(biases[i], db)
            src, vk = (x2, v0) if i == 0 else (ys[i - 1], (D * layer_size[i - 1], 1, layer_size[i - 1]))
            dhid = None
            if i > 0:
                dhid = _empty((B * D, h), x2)        # grad of the first h maps of layer i-1, [B, D, h]
            dw = _empty((kdim, size), x2)
            K.fill(dw, 0.0)
            for b0 in range(0, B, chunk):
                nb = min(chunk, B - b0)
                zc = z.reshape(-1)[:nb * D * kdim].reshape(nb * D, kdim)
                K.cin_outer_fwd(x2, v0, src, vk, zc, b0, nb, m, h, D)          # recompute Z (stays in L2)
                dzc = dz_[b0 * D:(b0 + nb) * D]
                K.gemm(zc, dzc, c=dw, trans_a=True, accumulate=True, precision=GEMM_PRECISION,
                       m=kdim, n=size, k=nb * D)
                dzf = K.gemm(dzc, ws[i], c=zc, trans_b=True, precision=GEMM_PRECISION, m=nb * D, n=kdim, k=size)
                if i == 0:
                    # X_k is X_0 itself: both factors accumulate into dx
                    K.cin_outer_bwd(dzf, x2, v0, src, vk, dx, gx, True, dx, gx, True, b0, nb, m, h, D)
                else:
                    K.cin_outer_bwd(dzf, x2, v0, src, vk, dx, gx, True, dhid, (D * h, 1, h), False, b0, nb,
                                    m, h, D)
            E.add_grad(filters[i], dw.reshape(filters[i].shape))
            dh = dhid
        E.add_grad(x, dx.reshape(x.shape))

    E.record([res], [x] + list(filters) + list(biases), bwd)
    return res


def interacting_attention(q, k, v, res, heads, dhead, scaling):
    """softmax(q_h k_h^T) v_h (+ res) -> relu, per sample and head (layers/interaction.py:760-777)."""
    B, F, HD = q.shape
    qt, kt, vt = E.contiguous(q), E.contiguous(k), E.contiguous(v)
    rt = E.contiguous(res) if res is not None else None
    out = K.interacting_fwd(qt, kt, vt, rt, B, F, heads, dhead, scaling)
    o = E.Var(out)

    def bwd(grads):
        g = grads[0]
        if not g.is_contiguous():
            g = g.contiguous()
        dq, dk, dv, dres = K.interacting_bwd(qt, kt, vt, out, g, res is not None, B, F, heads, dhead, scaling)
        E.add_grad(q, dq)
        E.add_grad(k, dk)
        E.add_grad(v, dv)
        if res is not None:
            E.add_grad(res, dres)

    E.record([o], [q, k, v, res], bwd)
    return o


# ==================================================================================================
# sequence operators
# ==================================================================================================
def din_att_input(query, keys):
    """[q, k, q-k, q*k] along the last axis (layers/core.py:98-101)."""
    B, T, Edim = keys.shape
    qt, ldq = query.flat2d()
    if qt is None:
        qt = E.contiguous(query).reshape(B, Edim)
        ldq = Edim
    kt, ldk = keys.flat2d()
    if kt is None:
        kt = E.contiguous(keys).reshape(B, T * Edim)
        ldk = T * Edim
    out = K.din_att_input_fwd(qt, ldq, kt, ldk, B, T, Edim)
    res = E.Var(out)

    def bwd(grads):
        g = grads[0]
        if not g.is_contiguous():
            g = g.contiguous()
        dq, dk = K.din_att_input_bwd(qt, ldq, kt, ldk, g, B, T, Edim)
        E.add_grad(query, dq.reshape(query.shape))
        E.add_grad(keys, dk.reshape(keys.shape))

    E.record([res], [query, keys], bwd)
    return res


def din_att_fusable(query, keys, n_out):
    """[q, k, q-k, q*k] can be generated inside the first attention GEMM (b2ctr_att_gemm)."""
    B, T, Edim = keys.shape
    return (GEMM_PRECISION == L.GEMM_BF16X3 and Edim % 8 == 0 and B * T >= 256 and n_out >= 8
            and n_out % 4 == 0)


def din_att_first(query, keys, w, b, activation):
    """act([q, k, q-k, q*k] @ w + b) -> [B, T, n] without materialising the [B, T, 4E] attention input
    (layers/core.py:96-103).  The backward pass generates the same operand again for the kernel gradient; only
    d(input) = dZ W^T exists in memory, to be folded back onto q and k."""
    B, T, Edim = keys.shape
    qt, ldq = query.flat2d()
    if qt is None or ldq % 4 or qt.data_ptr() % 16:
        qt = E.contiguous(query).reshape(B, Edim)
        ldq = Edim
    kt, ldk = keys.flat2d()
    if kt is None or ldk % 4 or kt.data_ptr() % 16:
        kt = E.contiguous(keys).reshape(B, T * Edim)
        ldk = T * Edim
    act = L.ACT_BY_NAME[activation]
    wd, bd = _wdata(w), (_wdata(b) if b is not None else None)
    n = wd.shape[1]
    wp = K.split_planes(wd)
    y = K.att_gemm(0, qt, ldq, kt, ldk, B, T, Edim, n, wp, bias=bd, act=act)
    out = E.Var(y.reshape(B, T, n))
    rows = B * T

    def bwd(grads):
        dy = grads[0].reshape(rows, n)
        if not dy.is_contiguous():
            dy = dy.contiguous()
        need_db = b is not None and b.requires_grad
        dzp = None
        if act != L.ACT_NONE or need_db:
            if act != L.ACT_NONE and K.planes_fusable(rows, n):
                dz, db, dzp = K.bias_act_bwd(dy, y, act, want_dz=True, want_dbias=need_db, want_planes=True)
            else:
                dz, db = K.bias_act_bwd(dy, y, act, want_dz=act != L.ACT_NONE, want_dbias=need_db)
            if dz is None:
                dz = dy
        else:
            dz, db = dy, None
        if dzp is None:
            dzp = K.split_planes(dz)
        if w.requires_grad:
            dw = K.att_gemm(1, qt, ldq, kt, ldk, B, T, Edim, n, dzp, split_k=_split_k(4 * Edim, n, rows))
            E.add_grad(w, dw)
        if need_db:
            E.add_grad(b, db)
        if query.requires_grad or keys.requires_grad:
            da = K.gemm(dz, wd, trans_b=True, precision=L.GEMM_BF16X3, m=rows, n=4 * Edim, k=n, a_planes=dzp, b_planes=wp)
            dq, dk = K.din_att_input_bwd(qt, ldq, kt, ldk, da, B, T, Edim)
            E.add_grad(query, dq.reshape(query.shape))
            E.add_grad(keys, dk.reshape(keys.shape))

    E.record([out], [query, keys, w, b], bwd)
    return out


def din_attention_pool(score, keys, mask_u8, weight_normalization, return_score):
    """masked fill -> [softmax] -> score @ keys   (layers/sequence.py:278-291)."""
    B, T, Edim = keys.shape
    st = E.contiguous(score).reshape(B, T)
    kt, ldk = keys.flat2d()
    if kt is None:
        kt = E.contiguous(keys).reshape(B, T * Edim)
        ldk = T * Edim
    out, w = K.din_pool_fwd(st, kt, ldk, mask_u8, B, T, Edim, weight_normalization, return_score)
    res = E.Var(out)

    def bwd(grads):
        g = grads[0]
        if not g.is_contiguous():
            g = g.contiguous()
        dscore, dkeys = K.din_pool_bwd(w, kt, ldk, mask_u8, g, B, T, Edim, weight_normalization, return_score,
                                       want_dkeys=keys.requires_grad)
        E.add_grad(score, dscore.reshape(score.shape))
        if dkeys is not None:
            E.add_grad(keys, dkeys.reshape(keys.shape))

    E.record([res], [score, keys], bwd)
    return res


def _len_i32(lengths):
    t = lengths.data
    if t.dtype != torch.int32:
        raise ValueError("sequence lengths must be int32")
    return dense_i32(t).reshape(-1)


def dense_i32(t):
    """Contiguous copy of a strided int32 [B, W] window through the copy2d kernel (bit-exact 4-byte moves)."""
    if t.is_contiguous():
        return t
    t2 = t.reshape(t.shape[0], -1) if t.dim() != 2 else t
    out = torch.empty(t2.shape, dtype=torch.int32, device=t.device)
    K.copy2d(t2.view(torch.float32), t2.stride(0), out.view(torch.float32), out.stride(0), t2.shape[0], t2.shape[1])
    return out


def seqpool(seq, mode, mask_u8=None, lengths=None):
    B, T, Edim = seq.shape
    xt = E.contiguous(seq)
    ln = _len_i32(lengths) if lengths is not None else None
    code = L.POOL_BY_NAME[mode]
    out = K.seqpool_fwd(xt, mask_u8, ln, B, T, Edim, code)
    res = E.Var(out)

    def bwd(grads):
        g = grads[0]
        if not g.is_contiguous():
            g = g.contiguous()
        E.add_grad(seq, K.seqpool_bwd(xt, mask_u8, ln, g, B, T, Edim, code))

    E.record([res], [seq], bwd)
    return res


def weighted_seq(seq, weights, normalize, mask_u8=None, lengths=None):
    B, T, Edim = seq.shape
    xt = E.contiguous(seq)
    wt_in = E.contiguous(weights).reshape(B, T)
    ln = _len_i32(lengths) if lengths is not None else None
    wt = K.seqweight(wt_in, mask_u8, ln, B, T, normalize)
    out = K.seqscale(xt, wt, B * T, Edim)
    res = E.Var(out, mask=seq.mask)

    def bwd(grads):
        g = grads[0]
        if not g.is_contiguous():
            g = g.contiguous()
        E.add_grad(seq, K.seqscale(g, wt, B * T, Edim))     # weights are inputs: no gradient needed

    E.record([res], [seq], bwd)
    return res


def _stats_for(x2, m, n, mean_w, var_w, training, momentum):
    if training:
        stats = K.colstats(x2, n, m, n)
        K.moving_update(mean_w.materialize(), stats[0], momentum)
        K.moving_update(var_w.materialize(), stats[1], momentum)
        return stats[0], stats[1]
    return mean_w.materialize(), var_w.materialize()


def dice(x, alphas, moving_mean, moving_var, eps, training, momentum=0.99):
    """Dice (layers/activation.py:59-64) over the last axis; batch statistics over all leading axes."""
    xt = E.contiguous(x)
    n = xt.shape[-1]
    m = xt.numel() // n
    x2 = xt.reshape(m, n)
    mean, var = _stats_for(x2, m, n, moving_mean, moving_var, training, momentum)
    al = alphas.materialize()
    y = K.dice_fwd(x2, mean, var, al, m, n, eps)
    res = E.Var(y.reshape(xt.shape))

    def bwd(grads):
        g = grads[0].reshape(m, n)
        if not g.is_contiguous():
            g = g.contiguous()
        dx, dalpha = K.dice_bwd(x2, mean, var, al, g, m, n, eps, training)
        E.add_grad(x, dx.reshape(x.shape))
        E.add_grad(alphas, dalpha)

    E.record([res], [x, alphas], bwd)
    return res


def batchnorm(x, gamma, beta, moving_mean, moving_var, eps, training, momentum=0.99):
    xt = E.contiguous(x)
    n = xt.shape[-1]
    m = xt.numel() // n
    x2 = xt.reshape(m, n)
    mean, var = _stats_for(x2, m, n, moving_mean, moving_var, training, momentum)
    gd = gamma.materialize() if gamma is not None else None
    bd = beta.materialize() if beta is not None else None
    y = K.bn_apply(x2, mean, var, gd, bd, m, n, eps)
    res = E.Var(y.reshape(xt.shape))

    def bwd(grads):
        g = grads[0].reshape(m, n)
        if not g.is_contiguous():
            g = g.contiguous()
        dx, dgamma, dbeta = K.bn_bwd(x2, mean, var, gd, g, m, n, eps, training)
        E.add_grad(x, dx.reshape(x.shape))
        if gamma is not None:
            E.add_grad(gamma, dgamma)
        if beta is not None:
            E.add_grad(beta, dbeta)

    E.record([res], [x, gamma, beta], bwd)
    return res


def mha(q, k, v, heads, scale, blinding=False, rate=0.0, seed=0, res=None, qlen=None, klen=None, qmask=None,
        kmask=None):
    """Masked multi-head scaled-dot-product attention of the reference's Transformer (layers/sequence.py:544-617)
    on [B, T, heads*d] projections, read in place through their row pitches; ``res`` (added in the epilogue) is
    the residual.  Validity from int32 lengths (Vars [B, 1]) or uint8 [B, T] masks.  Only [B, heads, T, 2]
    softmax statistics are kept for the backward, which recomputes the probabilities."""
    B, T, W = q.shape
    d = W // heads
    for name, x in (("k", k), ("v", v), ("res", res)):
        if x is not None and tuple(x.shape) != (B, T, W):
            raise ValueError("mha: %s has shape %s, the queries %s" % (name, tuple(x.shape), (B, T, W)))
    for name, x, want in (("qlen", qlen, B), ("klen", klen, B)):
        if x is not None and x.data.numel() != want:
            raise ValueError("mha: %s has %d entries for a batch of %d" % (name, x.data.numel(), want))
    for name, x in (("qmask", qmask), ("kmask", kmask)):
        if x is not None and tuple(x.shape) != (B, T):
            raise ValueError("mha: %s has shape %s, expected %s" % (name, tuple(x.shape), (B, T)))
    if rate:
        mark_uncapturable()
    q2, ldq = _as2d(q)
    k2, ldk = _as2d(k)
    v2, ldv = _as2d(v)
    r2, ldr = _as2d(res) if res is not None else (None, 0)
    ql = _len_i32(qlen) if qlen is not None else None
    kl = _len_i32(klen) if klen is not None else None
    kw = dict(blinding=blinding, rate=rate, seed=seed, qlen=ql, klen=kl, qmask=qmask, kmask=kmask)
    out, stats = K.mha_fwd(q2, ldq, k2, ldk, v2, ldv, B, T, heads, d, scale, res=r2, ldr=ldr, **kw)
    o = E.Var(out.reshape(B, T, W))

    def bwd(grads):
        g = grads[0].reshape(B * T, W)
        if not g.is_contiguous():
            g = g.contiguous()
        dq, dk, dv = K.mha_bwd(g, W, q2, ldq, k2, ldk, v2, ldv, stats, B, T, heads, d, scale, **kw)
        E.add_grad(q, dq.reshape(q.shape))
        E.add_grad(k, dk.reshape(k.shape))
        E.add_grad(v, dv.reshape(v.shape))
        if res is not None:
            E.add_grad(res, g.reshape(res.shape))

    E.record([o], [q, k, v, res], bwd)
    return o


def layernorm(a, gamma, beta, eps, b=None):
    """LayerNormalization over the last axis of a (+ b) (layers/normalization.py:34-43); the sum of the two
    summands is formed inside the kernel, and both receive the same gradient."""
    shape = a.shape
    n = shape[-1]
    a2, lda = _as2d(a)
    b2, ldb = _as2d(b) if b is not None else (None, 0)
    rows = a2.shape[0]
    gd = _wdata(gamma) if gamma is not None else None
    bd = _wdata(beta) if beta is not None else None
    y, stats = K.layernorm_fwd(a2, lda, b2, ldb, gd, bd, rows, n, eps)
    res = E.Var(y.reshape(shape))

    def bwd(grads):
        g = grads[0].reshape(rows, n)
        if not g.is_contiguous():
            g = g.contiguous()
        dx, dgamma, dbeta = K.layernorm_bwd(a2, lda, b2, ldb, gd, stats, g, rows, n,
                                            want_dgamma=gamma is not None and gamma.requires_grad,
                                            want_dbeta=beta is not None and beta.requires_grad)
        E.add_grad(a, dx.reshape(shape))
        if b is not None:
            # the same tensor for both summands: see ops.add on why the Transformer's tape order makes that safe
            E.add_grad(b, dx.reshape(shape))
        if dgamma is not None:
            E.add_grad(gamma, dgamma.reshape(gamma.shape))
        if dbeta is not None:
            E.add_grad(beta, dbeta.reshape(beta.shape))

    E.record([res], [a, b, gamma, beta], bwd)
    return res


def full_lengths(batch, T, device):
    """int32 [B, 1] filled with T (the unmasked sequence of reduce_mean / reduce_sum over the time axis), written
    by the fill kernel through a float32 view of the bits."""
    import struct
    out = torch.empty((batch, 1), dtype=torch.int32, device=device)
    K.fill(out.view(torch.float32), struct.unpack("<f", struct.pack("<i", int(T)))[0])
    return E.Var(out)


def dropout(x, rate, seed):
    mark_uncapturable()
    xt = E.contiguous(x)
    res = E.Var(K.dropout(xt, rate, seed))

    def bwd(grads):
        g = grads[0]
        if not g.is_contiguous():
            g = g.contiguous()
        E.add_grad(x, K.dropout(g, rate, seed))

    E.record([res], [x], bwd)
    return res


def reduce(x, kind, axis, keep_dims):
    """reduce_sum / reduce_mean / reduce_max shims of layers/utils.py:245-303 for the common cases."""
    if kind == "sum" and (axis in (-1, x.data.dim() - 1)) and x.data.dim() == 2:
        r = rowsum(x)
        return r if keep_dims else reshape(r, (x.shape[0],))
    shape = tuple(x.data.shape)
    if (kind == "sum" and x.data.dim() > 2 and axis in (-1, x.data.dim() - 1)
            and all(d == 1 for d in shape[1:-1])):
        # [B, 1.., E] over the last axis (ONN's K.sum(product, axis=-1), onn.py:96): the row sum of [B, E]
        r = rowsum(x)
        return reshape(r, shape[:-1] + ((1,) if keep_dims else ()))
    raise NotImplementedError("reduce_%s over axis %r of a %d-D tensor" % (kind, axis, x.data.dim()))


def multiply(xs):
    """Keras Multiply of same-shaped operands on b2ctr_ewise; d a_k = g * prod of the others."""
    if len(xs) != 2:
        return multiply([multiply(xs[:-1]), xs[-1]])
    a, b = xs
    if tuple(a.shape) != tuple(b.shape):
        raise ValueError("multiply: operands of shapes %s and %s differ" % (tuple(a.shape), tuple(b.shape)))
    at, bt = E.contiguous(a), E.contiguous(b)
    res = E.Var(K.ewise(0, at, bt))

    def bwd(grads):
        g = grads[0].reshape(at.shape).contiguous()
        if a.requires_grad:
            E.add_grad(a, K.ewise(0, g, bt))
        if b.requires_grad:
            E.add_grad(b, K.ewise(0, g, at))

    E.record([res], [a, b], bwd)
    return res


def div(x, y):
    raise NotImplementedError("div is only used inside SequencePoolingLayer, which has its own kernel")


def softmax(x, dim=-1, scale=1.0):
    """scale * softmax(x) along the last axis of a 2-D x (layers/utils.py:306-310; IFM's F * softmax(z, dim=1),
    ifm.py:60) on b2ctr_softmax_rows_fwd / _bwd.  Other ranks and axes: NotImplementedError."""
    if x.data.dim() != 2 or dim not in (-1, 1):
        raise NotImplementedError("softmax over axis %r of a %d-D tensor: only the last axis of a 2-D tensor is "
                                  "supported" % (dim, x.data.dim()))
    x2, _ = _as2d(x)
    scale = float(scale)
    y = K.softmax_rows_fwd(x2, scale)
    res = E.Var(y)

    def bwd(grads):
        g = grads[0].reshape(y.shape)
        if g.stride(1) != 1:
            g = g.contiguous()
        E.add_grad(x, K.softmax_rows_bwd(y, g, scale))

    E.record([res], [x], bwd)
    return res
