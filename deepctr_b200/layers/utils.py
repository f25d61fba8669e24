"""Host mirror of deepctr/layers/utils.py: Hash, Linear, Concat / NoMask / concat_func, add_func,
combined_dnn_input (reference lines cited per class)."""
import csv

import numpy as np
import torch

from .. import _lib as L
from .. import kernels as K
from .. import engine as E
from .. import ops
from ..engine import Layer, Flatten, Add, Zeros, glorot_normal, l2


class NoMask(Layer):
    """deepctr/layers/utils.py:26-38."""

    def call(self, x, mask=None, **kwargs):
        return x

    def compute_mask(self, inputs, mask=None):
        return None


# ---- Hash ----------------------------------------------------------------------------------------
_M64 = (1 << 64) - 1
_K0, _K1, _K2 = 0xc3a5c85c97cb3127, 0xb492b66fbe98f273, 0x9ae16a3b2f90404f


def _rot(v, s):
    return ((v >> s) | (v << (64 - s))) & _M64


def _hl16(u, v, mul):
    a = ((u ^ v) * mul) & _M64
    a ^= a >> 47
    b = ((v ^ a) * mul) & _M64
    b ^= b >> 47
    return (b * mul) & _M64


def _fingerprint64(s):
    """FarmHash Fingerprint64 for host-side STRING ids (<= 64 bytes); integer ids are hashed on the
    device by the gather kernel (csrc/embed.cu).  Published algorithm (google/farmhash); the product
    needs its own copy because oracle/ is test-only."""
    n = len(s)
    f64 = lambda i: int.from_bytes(s[i:i + 8], "little")
    f32 = lambda i: int.from_bytes(s[i:i + 4], "little")
    if n <= 16:
        if n >= 8:
            mul = (_K2 + n * 2) & _M64
            a = (f64(0) + _K2) & _M64
            b = f64(n - 8)
            c = (_rot(b, 37) * mul + a) & _M64
            d = ((_rot(a, 25) + b) * mul) & _M64
            return _hl16(c, d, mul)
        if n >= 4:
            mul = (_K2 + n * 2) & _M64
            return _hl16((n + (f32(0) << 3)) & _M64, f32(n - 4), mul)
        if n > 0:
            y = (s[0] + (s[n >> 1] << 8)) & 0xFFFFFFFF
            z = (n + (s[n - 1] << 2)) & 0xFFFFFFFF
            v = ((y * _K2) & _M64) ^ ((z * _K0) & _M64)
            return ((v ^ (v >> 47)) * _K2) & _M64
        return _K2
    mul = (_K2 + n * 2) & _M64
    if n <= 32:
        a = (f64(0) * _K1) & _M64
        b = f64(8)
        c = (f64(n - 8) * mul) & _M64
        d = (f64(n - 16) * _K2) & _M64
        return _hl16((_rot((a + b) & _M64, 43) + _rot(c, 30) + d) & _M64,
                     (a + _rot((b + _K2) & _M64, 18) + c) & _M64, mul)
    if n <= 64:
        a = (f64(0) * _K2) & _M64
        b = f64(8)
        c = (f64(n - 8) * mul) & _M64
        d = (f64(n - 16) * _K2) & _M64
        y = (_rot((a + b) & _M64, 43) + _rot(c, 30) + d) & _M64
        z = _hl16(y, (a + _rot((b + _K2) & _M64, 18) + c) & _M64, mul)
        e = (f64(16) * mul) & _M64
        f = f64(24)
        g = ((y + f64(n - 32)) * mul) & _M64
        h = ((z + f64(n - 24)) * mul) & _M64
        return _hl16((_rot((e + f) & _M64, 43) + _rot(g, 30) + h) & _M64,
                     (e + _rot((f + a) & _M64, 18) + g) & _M64, mul)
    raise NotImplementedError("string ids longer than 64 bytes are not supported")


def _as_bytes(v):
    if isinstance(v, bytes):
        return v
    if isinstance(v, str):
        return v.encode("utf-8")
    return str(int(v)).encode("ascii")


_vocab_cache = {}


def _load_vocabulary(path):
    """TextFileInitializer(path, 'string', 1, 'int64', 0, ','): key column 1, value column 0
    (deepctr/layers/utils.py:81-82)."""
    if path not in _vocab_cache:
        table = {}
        with open(path, newline="") as fh:
            for row in csv.reader(fh):
                if len(row) >= 2:
                    table[row[1].encode("utf-8")] = int(row[0])
        _vocab_cache[path] = table
    return _vocab_cache[path]


def host_hash_array(a, num_buckets, mask_zero=False, vocabulary_path=None, default_value=0):
    a = np.asarray(a)
    flat = a.reshape(-1)
    out = np.empty(flat.shape, dtype=np.int64)
    vocab = _load_vocabulary(vocabulary_path) if vocabulary_path else None
    nb = num_buckets - 1 if mask_zero else num_buckets
    cache = {}
    for i, v in enumerate(flat):
        s = _as_bytes(v.item() if hasattr(v, "item") else v)
        r = cache.get(s)
        if r is None:
            if vocab is not None:
                r = vocab.get(s, default_value)
            else:
                h = _fingerprint64(s) % nb
                r = (0 if s == b"0" else h + 1) if mask_zero else h
            cache[s] = r
        out[i] = r
    return out.reshape(a.shape)


class Hash(Layer):
    """deepctr/layers/utils.py:41-121.  Integer ids: FarmHash on the device (b2ctr_hash64, or inline in
    the fused gather when the planner folds this layer).  Strings / vocabulary files: host lookup."""

    def __init__(self, num_buckets, mask_zero=False, vocabulary_path=None, default_value=0, **kwargs):
        self.num_buckets = num_buckets
        self.mask_zero = mask_zero
        self.vocabulary_path = vocabulary_path
        self.default_value = default_value
        Layer.__init__(self, **kwargs)

    def _output_dtype(self, inputs):
        return "int64"

    def __call__(self, inputs, **kwargs):
        # eager convenience: accept raw python / numpy strings
        if not isinstance(inputs, (E.KTensor, E.Var)):
            a = np.asarray(inputs)
            if a.dtype.kind in ("U", "S", "O") or self.vocabulary_path:
                return host_hash_array(a, self.num_buckets, self.mask_zero, self.vocabulary_path,
                                       self.default_value)
        return Layer.__call__(self, inputs, **kwargs)

    def call(self, x, mask=None, **kwargs):
        if self.vocabulary_path:
            from .. import ops
            ops.mark_uncapturable()           # host-side vocabulary lookup: not CUDA-graph capturable
            ids = x.data.cpu().numpy()
            out = host_hash_array(ids, self.num_buckets, self.mask_zero, self.vocabulary_path, self.default_value)
            return E.Var(torch.from_numpy(out).to(x.data.device))
        return E.Var(K.hash64(x.data, self.num_buckets, self.mask_zero))

    def compute_output_shape(self, input_shape):
        return input_shape

    def get_config(self):
        config = {'num_buckets': self.num_buckets, 'mask_zero': self.mask_zero,
                  'vocabulary_path': self.vocabulary_path, 'default_value': self.default_value}
        base = Layer.get_config(self)
        return dict(list(base.items()) + list(config.items()))


# ---- Linear ----------------------------------------------------------------------------------------
class Linear(Layer):
    """deepctr/layers/utils.py:124-186.  Output is always [B,1] (mode 0 returns [B,1,1] in the
    reference; PredictionLayer reshapes to (-1,1) either way, core.py:257)."""

    def __init__(self, l2_reg=0.0, mode=0, use_bias=False, seed=1024, **kwargs):
        self.l2_reg = l2_reg
        if mode not in [0, 1, 2]:
            raise ValueError("mode must be 0,1 or 2")
        self.mode = mode
        self.use_bias = use_bias
        self.seed = seed
        Layer.__init__(self, **kwargs)

    def build(self, input_shape):
        if self.use_bias:
            self.bias = self.add_weight(name='linear_bias', shape=(1,), initializer=Zeros(), trainable=True)
        if self.mode == 1:
            self.kernel = self.add_weight('linear_kernel', shape=[int(input_shape[-1]), 1],
                                          initializer=glorot_normal(self.seed), regularizer=l2(self.l2_reg))
        elif self.mode == 2:
            self.kernel = self.add_weight('linear_kernel', shape=[int(input_shape[1][-1]), 1],
                                          initializer=glorot_normal(self.seed), regularizer=l2(self.l2_reg))
        self.built = True

    def call(self, inputs, **kwargs):
        if self.mode == 1:
            return ops.dense(ops.flatten(inputs), self.kernel, self.bias if self.use_bias else None)
        return self.combine(ops.rowsum(inputs if self.mode == 0 else inputs[0]), inputs)

    def combine(self, sparse_sum, inputs):
        """Modes 0 and 2: the output from ``sparse_sum`` [B, 1], the row-sum of the sparse input (computed here, or
        by the fused gather: inputs.EmbeddingPlanner._linear), plus the bias (mode 0) or the dense part (mode 2)."""
        bias = self.bias if self.use_bias else None
        if self.mode == 0:
            return sparse_sum if bias is None else ops.add_bias(sparse_sum, bias)
        fc = ops.dense(ops.flatten(inputs[1]), self.kernel, bias)
        return ops.add_n([sparse_sum, fc])

    def compute_output_shape(self, input_shape):
        return (None, 1)

    def compute_mask(self, inputs, mask=None):
        return None

    def get_config(self):
        config = {'mode': self.mode, 'l2_reg': self.l2_reg, 'use_bias': self.use_bias, 'seed': self.seed}
        base = Layer.get_config(self)
        return dict(list(base.items()) + list(config.items()))


class RefineWeight(Layer):
    """The Lambda of feature_column.py:193-200 (IFM / DIFM refine weights): the dim-1 linear lookups [B, 1, F_lin]
    times expand_dims(m, 1) for m [B, F] (b2ctr_field_scale_fwd with dim 1).  F_lin must equal F: the reference
    broadcasts when one of them is 1 and fails inside TensorFlow otherwise; here both are a ValueError at build time."""

    def build(self, input_shape):
        sparse, weight = input_shape
        if len(weight) != 2 or int(sparse[-1]) != int(weight[-1]):
            raise ValueError("sparse_feat_refine_weight has %s field weights but the linear part has %d sparse "
                             "features: the two counts must be equal" % (weight[-1], int(sparse[-1])))
        self.built = True

    def call(self, inputs, **kwargs):
        sparse, weight = inputs
        return ops.field_scale(sparse, weight)

    def compute_output_shape(self, input_shape):
        return input_shape[0]


class ZeroLogit(Layer):
    """feature_column.py:206-207: empty linear columns -> constant 0 logit."""

    def call(self, x, **kwargs):
        return ops.zeros_like_batch(x, 1)

    def compute_output_shape(self, input_shape):
        return (None, 1)


# ---- Concat ----------------------------------------------------------------------------------------
class Concat(Layer):
    """deepctr/layers/utils.py:189-233: concat whose mask is the AND of the input masks."""

    def __init__(self, axis, supports_masking=True, **kwargs):
        Layer.__init__(self, **kwargs)
        self.axis = axis
        self.supports_masking = supports_masking

    def call(self, inputs, **kwargs):
        return ops.concat(inputs, self.axis)

    def compute_mask(self, inputs, mask=None):
        if not self.supports_masking:
            return None
        if mask is None:
            return None
        if not isinstance(mask, list):
            raise ValueError('`mask` should be a list.')
        if not isinstance(inputs, list):
            raise ValueError('`inputs` should be a list.')
        if len(mask) != len(inputs):
            raise ValueError('The lists `inputs` and `mask` should have the same length.')
        if all(m is None for m in mask):
            return None
        out = None
        for m in mask:            # unmasked inputs contribute all-ones
            if m is not None:
                out = m if out is None else out.logical_and(m)
        return out

    def compute_output_shape(self, input_shape):
        shapes = [list(s) for s in input_shape]
        ax = self.axis if self.axis >= 0 else len(shapes[0]) + self.axis
        out = list(shapes[0])
        out[ax] = sum(s[ax] for s in shapes)
        return tuple(out)

    def get_config(self):
        config = {'axis': self.axis, 'supports_masking': self.supports_masking}
        base = Layer.get_config(self)
        return dict(list(base.items()) + list(config.items()))


def concat_func(inputs, axis=-1, mask=False):
    """deepctr/layers/utils.py:236-242."""
    if len(inputs) == 1:
        input = inputs[0]
        if not mask:
            input = NoMask()(input)
        return input
    return Concat(axis, supports_masking=mask)(inputs)


# ---- reductions exported by the reference (TF1/TF2 shims there; kernel wrappers here) --------------
def reduce_sum(input_tensor, axis=None, keep_dims=False, name=None, reduction_indices=None):
    return ops.reduce(input_tensor, "sum", axis, keep_dims)


def reduce_mean(input_tensor, axis=None, keep_dims=False, name=None, reduction_indices=None):
    return ops.reduce(input_tensor, "mean", axis, keep_dims)


def reduce_max(input_tensor, axis=None, keep_dims=False, name=None, reduction_indices=None):
    return ops.reduce(input_tensor, "max", axis, keep_dims)


def div(x, y, name=None):
    return ops.div(x, y)


def softmax(logits, dim=-1, name=None):
    return ops.softmax(logits, dim)


class _Add(Layer):
    """deepctr/layers/utils.py:313-325."""

    def call(self, inputs, **kwargs):
        if len(inputs) == 0:
            raise ValueError("_Add needs at least one input")
        return ops.add_n(inputs)

    def compute_output_shape(self, input_shape):
        best = input_shape[0]
        for s in input_shape[1:]:
            if len(s) > len(best):
                best = s
        return tuple(best)


def add_func(inputs):
    """deepctr/layers/utils.py:328-333."""
    if not isinstance(inputs, list):
        return inputs
    if len(inputs) == 1:
        return inputs[0]
    return _Add()(inputs)


class _CombinedDNNInput(Layer):
    """Flatten(concat(embeddings)) || Flatten(concat(dense)) as ONE op: when the embeddings are the
    planner's main buffer the dense features are appended behind them in place and the result is a
    zero-copy window (the K-padded GEMM operand; inputs.EmbeddingPlanner._combined_dnn_input)."""

    def call(self, inputs, **kwargs):
        return ops.concat(inputs, -1)

    def compute_output_shape(self, input_shape):
        return (input_shape[0][0], input_shape[0][1] + input_shape[1][1])


def combined_dnn_input(sparse_embedding_list, dense_value_list):
    """deepctr/layers/utils.py:336-346."""
    if len(sparse_embedding_list) > 0 and len(dense_value_list) > 0:
        sparse_dnn_input = Flatten()(concat_func(sparse_embedding_list))
        dense_dnn_input = Flatten()(concat_func(dense_value_list))
        return _CombinedDNNInput()([sparse_dnn_input, dense_dnn_input])
    elif len(sparse_embedding_list) > 0:
        return Flatten()(concat_func(sparse_embedding_list))
    elif len(dense_value_list) > 0:
        return Flatten()(concat_func(dense_value_list))
    else:
        raise NotImplementedError("dnn_feature_columns can not be empty list")
