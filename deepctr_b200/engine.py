"""Host-side runtime of the H100 CTR path.

What the reference gets from TensorFlow/Keras (symbolic ``Input``s, the ``Layer`` protocol, the
functional ``Model`` with compile/fit/predict, automatic differentiation, optimizers) is provided
here in ~one file, so that builders with the reference's signatures (deepctr_b200/models/) and layers with
its Keras protocol (deepctr_b200/layers/) have a runtime:

* ``Var``      - a device buffer (torch tensor used purely as memory handle) + gradient + Keras mask.
                 A Var can be a column WINDOW of a wider per-sample buffer (``base``/``col0``) - that is
                 how per-feature embeddings, their concatenation and the DNN input alias one HBM
                 buffer written once by the fused gather.
* ``Tape``     - reverse-mode tape; every op pushes a closure that launches the backward kernels.
* ``KTensor`` / ``Layer`` / ``Input`` / ``Model`` - the Keras functional surface (deepctr/layers/*.py
                 implement build / call / compute_output_shape / compute_mask / get_config against it).

All arithmetic is done by libb2ctr.so through ``kernels.py``; nothing here computes with torch.
"""
import gc
import inspect
import threading
from collections import OrderedDict

import os

import numpy as np
import torch

from . import _lib as L
from . import kernels as K

# ================================================================================================
# device / runtime tensors
# ================================================================================================


def device():
    if not torch.cuda.is_available():
        raise L.B2ctrError("deepctr_b200 needs a CUDA device (H100, sm_90a): the compute path has no "
                           "CPU fallback")
    return torch.device("cuda", torch.cuda.current_device())


class Var(object):
    """Runtime tensor.  ``data`` has the logical shape; when ``base`` is set, ``data`` is a strided
    window [col0, col0+ncols) of ``base.data`` (a [B, ld] buffer) and gradients are routed there."""
    __slots__ = ("data", "grad", "requires_grad", "mask", "base", "col0", "ncols", "owner", "name",
                 "vshape", "planes")

    def __init__(self, data, requires_grad=False, mask=None, base=None, col0=0, ncols=0, owner=None,
                 name=None, vshape=None):
        self.data = data
        self.planes = None      # (key, bf16 hi/lo planes) cache of ops.dense in BF16X3 mode
        self.vshape = vshape    # logical shape of a VIRTUAL var (data is None: fused away this step)
        self.grad = None
        self.requires_grad = requires_grad
        self.mask = mask
        self.base = base
        self.col0 = col0
        self.ncols = ncols
        self.owner = owner
        self.name = name

    @property
    def shape(self):
        return tuple(self.data.shape) if self.data is not None else tuple(self.vshape)

    def alias(self):
        v = Var(self.data, self.requires_grad, self.mask, self.base, self.col0, self.ncols, self.owner,
                vshape=self.vshape)
        if self.base is None:
            v.base, v.col0, v.ncols = self, 0, -1   # whole-tensor alias: grads flow to the original
        return v

    # ---- 2-D addressing used by every kernel wrapper --------------------------------------------
    def rows(self):
        return self.data.shape[0] if self.data.dim() > 0 else 1

    def as2d(self):
        """(tensor2d, ld): a [rows, cols] row-major window, rows = product of leading dims."""
        t = self.data
        if t.dim() == 2:
            return t, t.stride(0)
        if t.dim() == 1:
            return t.unsqueeze(1), 1
        if t.is_contiguous():
            t2 = t.reshape(-1, t.shape[-1])
            return t2, t2.stride(0)
        # [B, 1.., C] strided window: collapse the unit dims
        if all(s == 1 for s in t.shape[1:-1]) and t.stride(-1) == 1:
            t2 = t.as_strided((t.shape[0], t.shape[-1]), (t.stride(0), 1))
            return t2, t2.stride(0)
        return None, None

    def flat2d(self):
        """Per-sample flattening [B, prod(rest)] as a window (ld may exceed the width)."""
        t = self.data
        b = t.shape[0]
        w = int(np.prod(t.shape[1:])) if t.dim() > 1 else 1
        if t.is_contiguous():
            return t.reshape(b, w), w
        if t.dim() >= 2 and t.stride(-1) == 1:
            # window of a wider buffer: the non-batch dims must be dense among themselves
            exp = 1
            ok = True
            for d in range(t.dim() - 1, 0, -1):
                if t.shape[d] != 1 and t.stride(d) != exp:
                    ok = False
                    break
                exp *= t.shape[d]
            if ok:
                return t.as_strided((b, w), (t.stride(0), 1)), t.stride(0)
        return None, None


def contiguous(var):
    """Return a dense copy (via the copy2d kernel) if ``var`` is a strided window."""
    t = var.data
    if t.is_contiguous():
        return t
    src, ld = var.flat2d()
    if src is None:
        raise L.B2ctrError("unsupported strided layout %s / %s" % (tuple(t.shape), tuple(t.stride())))
    out = torch.empty(t.shape, dtype=t.dtype, device=t.device)
    w = src.shape[1]
    K.copy2d(src, ld, out, w, src.shape[0], w)
    return out


class _TapeNode(object):
    __slots__ = ("outputs", "backward", "tag", "keep")

    def __init__(self, outputs, backward, keep=False):
        self.outputs = outputs
        self.backward = backward
        self.tag = K.PROFILE_TAG       # bench attribution: the backward launches join the forward's group
        self.keep = keep               # the outputs' gradients are only read: an earlier node consumes them


class Tape(object):
    """Reverse-mode tape.  ``opt`` carries what fused backward kernels need (embedding lr ...)."""

    def __init__(self):
        self.nodes = []
        self.ctx = {}

    def record(self, outputs, backward, keep=False):
        self.nodes.append(_TapeNode(list(outputs), backward, keep))

    def backward(self):
        _state.opt_ctx = self.ctx
        try:
            for node in reversed(self.nodes):
                grads = [o.grad for o in node.outputs]
                if all(g is None for g in grads):
                    continue
                if node.tag is not None and K.PROFILE is not None:
                    with K.profile_tag(node.tag):
                        node.backward(grads)
                else:
                    node.backward(grads)
                if not node.keep:
                    for o in node.outputs:
                        o.grad = None   # free as we go
        finally:
            _state.opt_ctx = None
        self.nodes = []


_state = threading.local()


def current_tape():
    return getattr(_state, "tape", None)


def current_opt():
    """Context of the running backward pass (optimizer for fused embedding updates)."""
    return getattr(_state, "opt_ctx", None)


class KMask(object):
    """A Keras mask kept symbolic until a kernel needs it: the AND of ``id != 0`` terms (Embedding
    mask_zero, layers/utils.py:198-228 for the AND across concatenated features) and/or ``t < len``."""

    def __init__(self, ids=None, hashed=None, lengths=None, maxlen=None):
        self.terms = [(t, hashed) for t in (ids or [])]
        self.lengths, self.maxlen = lengths, maxlen
        self._u8 = None

    def logical_and(self, other):
        if other is None:
            return self
        m = KMask()
        m.terms = self.terms + other.terms
        m.lengths = self.lengths if self.lengths is not None else other.lengths
        m.maxlen = self.maxlen if self.maxlen is not None else other.maxlen
        return m

    def materialize(self):
        """uint8 [B, T] on the device (1 = valid)."""
        if self._u8 is not None:
            return self._u8
        out = None
        if self.lengths is not None:
            ln = self.lengths
            if not ln.is_contiguous():
                from . import ops
                ln = ops.dense_i32(ln.reshape(ln.shape[0], -1)).reshape(-1)
            out = K.mask_from_len(ln, self.maxlen)
        for ids, hashed in self.terms:
            t = ids.reshape(ids.shape[0], -1)
            if not t.is_contiguous():
                if t.dtype == torch.int32:
                    from . import ops
                    t = ops.dense_i32(t)
                else:
                    t = t.contiguous()
            if hashed is not None and hashed[0] == L.HASH_FARM:
                raise L.B2ctrError("mask of a hashed feature without mask_zero is not defined by the reference")
            out = K.mask_nonzero_and(t, out)
        self._u8 = out
        return out


class recording(object):
    def __init__(self, tape):
        self.tape = tape

    def __enter__(self):
        self.prev = current_tape()
        _state.tape = self.tape
        return self.tape

    def __exit__(self, *a):
        _state.tape = self.prev


def record(outputs, inputs, backward, keep_grads=False):
    """Register a backward closure if a tape is active and any input needs a gradient.  ``keep_grads``: the
    closure only reads its outputs' gradients and leaves them for the node that produced those outputs (an op that
    wrote its result into a window of another op's buffer, see ops.fefm)."""
    tape = current_tape()
    if tape is None:
        return False
    if not any(v is not None and v.requires_grad for v in inputs):
        return False
    for o in outputs:
        o.requires_grad = True
    tape.record(outputs, backward, keep_grads)
    return True


def add_grad(var, g):
    """Accumulate gradient tensor ``g`` (logical shape of ``var``) into ``var``."""
    if var is None or not var.requires_grad or g is None:
        return
    if var.base is not None:
        base = var.base
        if var.ncols == -1:            # whole-tensor alias
            add_grad(base, g.reshape(base.data.shape) if g.shape != base.data.shape else g)
            return
        bt = base.data                  # [B, ld] buffer
        g2 = g.reshape(g.shape[0], -1)
        if base.grad is None:
            used = base.ncols if base.ncols > 0 else bt.shape[1]
            if (var.col0 == 0 and g2.shape[1] >= used and g2.stride(0) == bt.stride(0)
                    and g2.stride(1) == 1):
                # the window covers every used column and g was written with the buffer's ld
                # (ops.dense does that): adopt it, no zero-fill + accumulate pass
                base.grad = torch.as_strided(g2, tuple(bt.shape), tuple(bt.stride()), g2.storage_offset())
                base.requires_grad = True
                return
            base.grad = torch.empty_like(bt)
            K.fill(base.grad, 0.0)
        K.copy2d(g2, g2.stride(0), base.grad, base.grad.stride(0), g2.shape[0], var.ncols,
                 accumulate=True, dst_off=var.col0)
        return
    if var.grad is None:
        var.grad = g
    else:
        K.axpy(g.contiguous() if not g.is_contiguous() else g, var.grad, 1.0)


# ================================================================================================
# weights and initializers
# ================================================================================================
class Initializer(object):
    def host(self, shape):
        raise NotImplementedError

    def get_config(self):
        return {}


class Zeros(Initializer):
    def host(self, shape):
        return np.zeros(shape, dtype=np.float32)


class Ones(Initializer):
    def host(self, shape):
        return np.ones(shape, dtype=np.float32)


class Constant(Initializer):
    def __init__(self, value=0.0):
        self.value = value

    def host(self, shape):
        return np.full(shape, self.value, dtype=np.float32)


class RandomNormal(Initializer):
    """tf.keras.initializers.RandomNormal.  Large tables are initialised ON DEVICE by the Philox
    kernel (b2ctr_init_normal); small ones on the host with numpy (the TF RNG stream itself is not
    reproducible outside TF - parity tests always load explicit weights)."""

    def __init__(self, mean=0.0, stddev=0.05, seed=None):
        self.mean, self.stddev, self.seed = mean, stddev, seed

    def host(self, shape):
        rng = np.random.RandomState(self.seed)
        return rng.normal(self.mean, self.stddev, size=shape).astype(np.float32)

    def get_config(self):
        return {"mean": self.mean, "stddev": self.stddev, "seed": self.seed}


class TruncatedNormal(RandomNormal):
    def host(self, shape):
        rng = np.random.RandomState(self.seed)
        v = rng.normal(self.mean, self.stddev, size=shape)
        bad = np.abs(v - self.mean) > 2 * self.stddev
        while bad.any():
            v[bad] = rng.normal(self.mean, self.stddev, size=int(bad.sum()))
            bad = np.abs(v - self.mean) > 2 * self.stddev
        return v.astype(np.float32)


def _fans(shape):
    if len(shape) < 1:
        return 1, 1
    if len(shape) == 1:
        return shape[0], shape[0]
    rf = int(np.prod(shape[:-2])) if len(shape) > 2 else 1
    return shape[-2] * rf, shape[-1] * rf


class GlorotNormal(Initializer):
    def __init__(self, seed=None):
        self.seed = seed

    def host(self, shape):
        fi, fo = _fans(shape)
        std = np.sqrt(2.0 / (fi + fo)) / 0.87962566103423978
        return TruncatedNormal(0.0, std, self.seed).host(shape)


class GlorotUniform(Initializer):
    def __init__(self, seed=None):
        self.seed = seed

    def host(self, shape):
        fi, fo = _fans(shape)
        lim = np.sqrt(6.0 / (fi + fo))
        return np.random.RandomState(self.seed).uniform(-lim, lim, size=shape).astype(np.float32)


glorot_normal = GlorotNormal
glorot_uniform = GlorotUniform
_DEVICE_INIT_THRESHOLD = 1 << 22   # elements: above this, RandomNormal runs on the GPU


class l2(object):
    """tf.keras.regularizers.l2: penalty l2 * sum(w^2)."""

    def __init__(self, l2=0.01):
        self.l2 = float(l2) if l2 else 0.0


class Weight(Var):
    """A named parameter.  Materialised lazily so that graph construction (and the CPU test-suite)
    never needs a device; ``value()`` / ``set_value`` move it explicitly."""
    __slots__ = ("shape_", "initializer", "regularizer", "trainable", "host_value", "opt_state",
                 "sparse_grad")

    def __init__(self, name, shape, initializer=None, regularizer=None, trainable=True):
        Var.__init__(self, None, requires_grad=trainable, name=name)
        self.shape_ = tuple(int(s) for s in shape)
        self.initializer = initializer or Zeros()
        self.regularizer = regularizer
        self.trainable = trainable
        self.host_value = None
        self.opt_state = {}
        self.sparse_grad = False    # True: embedding table updated by the fused scatter, no .grad

    @property
    def shape(self):
        return self.shape_

    @property
    def l2(self):
        return self.regularizer.l2 if isinstance(self.regularizer, l2) else 0.0

    def numel(self):
        return int(np.prod(self.shape_)) if self.shape_ else 1

    def materialize(self):
        """Ensure ``data`` lives on the device."""
        if self.data is not None:
            return self.data
        dev = device()
        if self.host_value is not None:
            self.data = torch.from_numpy(np.ascontiguousarray(self.host_value)).to(dev)
            self.host_value = None
        elif (isinstance(self.initializer, RandomNormal) and type(self.initializer) is RandomNormal
              and self.numel() >= _DEVICE_INIT_THRESHOLD):
            self.data = torch.empty(self.shape_, dtype=torch.float32, device=dev)
            import zlib
            seed = self.initializer.seed if self.initializer.seed is not None else 0
            shard = self.opt_state.get("shard", (0, 1, 0))[0]
            K.init_normal(self.data, self.initializer.mean, self.initializer.stddev,
                          (seed * 0x9E3779B97F4A7C15 + zlib.crc32(self.name.encode()) * 1000003 + shard)
                          & 0xFFFFFFFFFFFFFFFF)
        else:
            self.data = torch.from_numpy(self.initializer.host(self.shape_)).to(dev)
        return self.data

    def value(self):
        """numpy copy (host).  Works without a GPU as long as the weight never went to the device."""
        if self.data is not None:
            return self.data.detach().cpu().numpy()
        if self.host_value is None:
            self.host_value = self.initializer.host(self.shape_)
        return np.array(self.host_value, copy=True)

    def set_value(self, arr):
        arr = np.asarray(arr, dtype=np.float32)
        if tuple(arr.shape) != self.shape_:
            raise ValueError("Weight %s expects shape %s, got %s" % (self.name, self.shape_, arr.shape))
        if self.data is not None:
            self.data.copy_(torch.from_numpy(np.ascontiguousarray(arr)))
        else:
            self.host_value = np.array(arr, copy=True)


# ================================================================================================
# symbolic graph (Keras functional API)
# ================================================================================================
class TensorShape(tuple):
    """Static shape of a KTensor: a tuple that also answers TensorFlow's ``as_list()`` (the reference's builders
    call ``tensor.get_shape().as_list()``, e.g. deepctr/models/sequence/bst.py:86)."""

    def as_list(self):
        return list(self)


class KTensor(object):
    """Symbolic tensor produced by ``Input`` or by calling a Layer on symbolic tensors."""
    _count = 0

    def __init__(self, shape, dtype="float32", node=None, index=0, name=None):
        self.shape = tuple(shape)
        self.dtype = dtype
        self.node = node
        self.index = index
        KTensor._count += 1
        self.name = name or "tensor_%d" % KTensor._count

    def get_shape(self):
        return TensorShape(self.shape)

    def __repr__(self):
        return "<KTensor %s shape=%s dtype=%s>" % (self.name, self.shape, self.dtype)


class Node(object):
    __slots__ = ("layer", "inputs", "kwargs", "outputs")

    def __init__(self, layer, inputs, kwargs):
        self.layer, self.inputs, self.kwargs, self.outputs = layer, inputs, kwargs, None


def _flatten(x):
    if isinstance(x, (list, tuple)):
        out = []
        for e in x:
            out.extend(_flatten(e))
        return out
    return [x]


def _map_structure(fn, x):
    if isinstance(x, (list, tuple)):
        return [_map_structure(fn, e) for e in x]
    return fn(x)


def _shape_of(x):
    return _map_structure(lambda t: tuple(t.shape), x)


_name_counts = {}


def clear_session():
    """tf.keras.backend.clear_session(): reset the per-class counters behind automatic layer names, so the
    next model built in this process is named like the first one (``dnn``, ``dense``, ``dense_1`` ...)."""
    _name_counts.clear()


def _snake_case(cls):
    """Keras' automatic layer name for a class (``DNN`` -> ``dnn``, ``CrossNet`` -> ``cross_net``,
    ``_Add`` -> ``private__add``): weight names ``<layer>/<weight>`` then line up with the reference's."""
    import re
    s = re.sub("(.)([A-Z][a-z0-9]+)", r"\1_\2", cls)
    s = re.sub("([a-z])([A-Z])", r"\1_\2", s).lower()
    return "private" + s if s.startswith("_") else s


def _auto_name(cls):
    base = _snake_case(cls)
    n = _name_counts.get(base, 0)
    _name_counts[base] = n + 1
    return base if n == 0 else "%s_%d" % (base, n)


def to_var(x):
    """Wrap user data (numpy / torch / Var) for eager layer calls."""
    if isinstance(x, Var):
        return x
    if isinstance(x, np.ndarray):
        x = torch.from_numpy(np.ascontiguousarray(x))
    if isinstance(x, torch.Tensor):
        if x.dtype == torch.float64:
            x = x.float()
        return Var(x.to(device()))
    raise TypeError("cannot convert %r to a device tensor" % type(x))


class Layer(object):
    """The Keras ``Layer`` contract the reference's operators implement (SURVEY.md section 8b):
    ``__init__(**hyper) / build(input_shape) / call(inputs, mask=None, training=None) /
    compute_output_shape / compute_mask / get_config``."""

    def __init__(self, name=None, trainable=True, dtype=None, **kwargs):
        self.name = name or _auto_name(self.__class__.__name__)
        self.trainable = trainable
        self.built = False
        self._weights = []
        self._sublayers = []
        if not hasattr(self, "supports_masking"):
            self.supports_masking = False
        self._call_args = None

    # ---- weights -------------------------------------------------------------------------------
    def add_weight(self, name=None, shape=(), initializer=None, regularizer=None, trainable=True,
                   dtype=None):
        if isinstance(initializer, type):
            initializer = initializer()
        w = Weight("%s/%s" % (self.name, name), shape, initializer, regularizer,
                   trainable and self.trainable)
        self._weights.append(w)
        return w

    def _track(self, layer):
        """Register a nested layer (its weights are addressed ``<this layer>/<attribute path>/<weight>``).
        Keras draws automatic names from one counter per class whether a layer is nested or not, so the
        nested layer consumes its class' next name too: in DIN the attention unit's inner DNN takes ``dnn``
        and the tower's DNN is ``dnn_1``, as in the reference."""
        _auto_name(layer.__class__.__name__)
        self._sublayers.append(layer)
        return layer

    @property
    def weights(self):
        ws = list(self._weights)
        for sl in self._sublayers:
            ws.extend(sl.weights)
        return ws

    @property
    def trainable_weights(self):
        return [w for w in self.weights if w.trainable]

    def get_weights(self):
        return [w.value() for w in self.weights]

    def set_weights(self, values):
        ws = self.weights
        if len(ws) != len(values):
            raise ValueError("layer %s has %d weights, got %d arrays" % (self.name, len(ws), len(values)))
        for w, v in zip(ws, values):
            w.set_value(v)

    # ---- protocol defaults ---------------------------------------------------------------------
    def build(self, input_shape):
        self.built = True

    def call(self, inputs, **kwargs):
        return inputs

    def compute_output_shape(self, input_shape):
        return input_shape

    def compute_mask(self, inputs, mask=None):
        if not self.supports_masking:
            return None
        return mask

    def get_config(self):
        return {"name": self.name, "trainable": self.trainable}

    @classmethod
    def from_config(cls, config):
        return cls(**config)

    # ---- invocation ----------------------------------------------------------------------------
    def _maybe_build(self, input_shape):
        if not self.built:
            self.build(input_shape)
            self.built = True

    def __call__(self, inputs, **kwargs):
        flat = _flatten(inputs)
        if any(isinstance(t, KTensor) for t in flat):
            if not all(isinstance(t, KTensor) for t in flat):
                raise TypeError("layer %s called with a mix of symbolic and concrete inputs" % self.name)
            in_shape = _shape_of(inputs)
            self._maybe_build(in_shape)
            out_shape = self.compute_output_shape(in_shape)
            node = Node(self, inputs, kwargs)
            dtype = self._output_dtype(inputs)
            if isinstance(out_shape, list) and out_shape and isinstance(out_shape[0], (list, tuple)):
                outs = [KTensor(s, dtype, node, i) for i, s in enumerate(out_shape)]
                node.outputs = outs
                return outs
            out = KTensor(tuple(out_shape), dtype, node, 0)
            node.outputs = [out]
            return out
        # eager: concrete data
        vars_in = _map_structure(to_var, inputs)
        self._maybe_build(_shape_of(vars_in))
        return self._invoke(vars_in, kwargs.get("training", False), kwargs)

    def _output_dtype(self, inputs):
        return "float32"

    # True on layers whose call() takes an ops.ScaledFields (the refine product kept as its factors) as it is; every
    # other layer receives the materialised product
    takes_scaled_fields = False

    def _invoke(self, vars_in, training, kwargs=None):
        if not self.takes_scaled_fields:
            vars_in = _concrete(vars_in)
        if self._call_args is None:
            try:
                self._call_args = set(inspect.signature(self.call).parameters)
            except (TypeError, ValueError):
                self._call_args = set()
        kw = {}
        masks = _map_structure(lambda v: v.mask, vars_in)
        if "mask" in self._call_args:
            has = any(m is not None for m in _flatten(masks))
            kw["mask"] = masks if has else None
        if "training" in self._call_args:
            kw["training"] = training
        out = self.call(vars_in, **kw)
        # attach the Keras mask the layer declares for its output
        if isinstance(out, Var):
            flat_in = _flatten(vars_in)
            if any(out is v for v in flat_in):
                out = out.alias()
            has = any(m is not None for m in _flatten(masks))
            out.mask = self.compute_mask(vars_in, masks if has else None)
        return out


def _concrete(vars_in):
    """``vars_in`` with every ops.ScaledFields replaced by its product (computed once), as call() receives it."""
    return _map_structure(lambda v: v.product() if isinstance(v, ops.ScaledFields) else v, vars_in)


class InputLayer(Layer):
    def __init__(self, shape, dtype="float32", name=None):
        Layer.__init__(self, name=name)
        self.shape = tuple(shape)
        self.dtype = dtype
        self.built = True


def Input(shape=None, name=None, dtype="float32", batch_shape=None, **kwargs):
    """tf.keras.layers.Input: a symbolic placeholder of shape (None,) + shape."""
    if isinstance(shape, int):
        shape = (shape,)
    if batch_shape is not None:
        full = tuple(batch_shape)
    else:
        full = (None,) + tuple(shape)
    layer = InputLayer(full, dtype, name=name)
    node = Node(layer, [], {})
    t = KTensor(full, dtype, node, 0, name=layer.name)
    node.outputs = [t]
    return t


# ================================================================================================
# plain Keras layers the builders import (Dense / Flatten / Concatenate / Lambda / Add)
# ================================================================================================
from . import ops  # noqa: E402  (ops needs Var / record defined above)


class Dense(Layer):
    """tf.keras.layers.Dense (used as ``Dense(1, use_bias=False)`` by every builder)."""

    def __init__(self, units, activation=None, use_bias=True, kernel_initializer=None,
                 kernel_regularizer=None, **kwargs):
        Layer.__init__(self, **kwargs)
        self.units, self.activation, self.use_bias = units, activation, use_bias
        self.kernel_initializer = kernel_initializer or GlorotUniform()
        self.kernel_regularizer = kernel_regularizer

    def build(self, input_shape):
        self.kernel = self.add_weight("kernel", (int(input_shape[-1]), self.units),
                                      self.kernel_initializer, self.kernel_regularizer)
        self.bias = self.add_weight("bias", (self.units,), Zeros()) if self.use_bias else None
        self.built = True

    def call(self, inputs, **kwargs):
        return ops.dense(inputs, self.kernel, self.bias, self.activation)

    def compute_output_shape(self, input_shape):
        return tuple(input_shape[:-1]) + (self.units,)

    def get_config(self):
        c = Layer.get_config(self)
        c.update(units=self.units, activation=self.activation, use_bias=self.use_bias)
        return c



def _pair(v, what):
    if isinstance(v, int):
        return (v, v)
    v = tuple(int(i) for i in v)
    if len(v) != 2:
        raise ValueError("%s must be an int or a pair, got %r" % (what, v))
    return v


class Conv2D(Layer):
    """tf.keras.layers.Conv2D as CCPM uses it (deepctr/models/ccpm.py:65-66): a kernel (width, 1) over [B, rows, E, C]
    channels_last, strides (1, 1), padding 'same', an activation of the package's set and a bias.  Each embedding
    coordinate is an independent 1-D signal over the rows; the layer is one stage of b2ctr_conv_stack, and in CCPM
    the planner (inputs.ConvStackPlan) runs every Conv2D and KMaxPooling of the stack in one launch.  Weights
    ``kernel`` [width, 1, C, filters] (glorot_uniform) and ``bias`` [filters] (zeros), as Keras names them.  Any
    other configuration raises NotImplementedError naming the argument."""

    def __init__(self, filters, kernel_size, strides=(1, 1), padding='valid', data_format=None, dilation_rate=(1, 1),
                 activation=None, use_bias=True, kernel_initializer=None, bias_initializer=None,
                 kernel_regularizer=None, bias_regularizer=None, **kwargs):
        from .layers.activation import fusable_activation
        ks = _pair(kernel_size, "kernel_size")
        if ks[1] != 1:
            raise NotImplementedError("Conv2D kernel_size %r: only (width, 1) kernels are supported" % (kernel_size,))
        if _pair(strides, "strides") != (1, 1):
            raise NotImplementedError("Conv2D strides %r: only (1, 1) is supported" % (strides,))
        if str(padding).lower() != "same":
            raise NotImplementedError("Conv2D padding %r: only 'same' is supported" % (padding,))
        if data_format not in (None, "channels_last"):
            raise NotImplementedError("Conv2D data_format %r: only 'channels_last' is supported" % (data_format,))
        if _pair(dilation_rate, "dilation_rate") != (1, 1):
            raise NotImplementedError("Conv2D dilation_rate %r: only (1, 1) is supported" % (dilation_rate,))
        if activation not in (None, "linear") and (not fusable_activation(activation) or activation == "dice"):
            raise NotImplementedError("Conv2D activation %r: only None, linear, relu, sigmoid and tanh are supported"
                                      % (activation,))
        if kernel_regularizer is not None or bias_regularizer is not None:
            raise NotImplementedError("Conv2D kernel_regularizer / bias_regularizer are not supported")
        Layer.__init__(self, **kwargs)
        self.filters, self.kernel_size, self.activation, self.use_bias = int(filters), ks, activation, use_bias
        self.kernel_initializer = kernel_initializer or GlorotUniform()
        self.bias_initializer = bias_initializer or Zeros()

    def build(self, input_shape):
        if len(input_shape) != 4:
            raise ValueError("Conv2D expects a 4-D input [batch, rows, embedding, channels], got %s"
                             % (tuple(input_shape),))
        rows, channels = int(input_shape[1]), int(input_shape[3])
        K.conv_stack_check(rows, channels, [("conv", self.kernel_size[0], self.filters)])
        self.kernel = self.add_weight("kernel", (self.kernel_size[0], 1, channels, self.filters),
                                      self.kernel_initializer)
        self.bias = self.add_weight("bias", (self.filters,), self.bias_initializer) if self.use_bias else None
        self.built = True

    def stage(self):
        """This layer as a b2ctr_conv_stack stage (ops.conv_stack)."""
        return ("conv", self.kernel_size[0], self.filters, self.activation, self.kernel, self.bias)

    def call(self, inputs, **kwargs):
        b, rows, dim, channels = inputs.data.shape
        return ops.conv_stack(inputs, [self.stage()], rows, dim, channels, (b, rows, dim, self.filters))

    def compute_output_shape(self, input_shape):
        return tuple(input_shape[:3]) + (self.filters,)

    def get_config(self):
        c = Layer.get_config(self)
        c.update(filters=self.filters, kernel_size=self.kernel_size, strides=(1, 1), padding="same",
                 activation=self.activation, use_bias=self.use_bias)
        return c

class Flatten(Layer):
    def call(self, inputs, **kwargs):
        return ops.flatten(inputs)

    def compute_output_shape(self, input_shape):
        n = 1
        for s in input_shape[1:]:
            n *= s
        return (input_shape[0], n)


class Reshape(Layer):
    """Keras' Reshape(target_shape): the per-sample shape becomes ``target_shape`` (one entry may be -1).  A window
    of a wider buffer stays a zero-copy view of it (PNN's linear_signal over the gather buffer)."""

    def __init__(self, target_shape, **kwargs):
        Layer.__init__(self, **kwargs)
        self.target_shape = tuple(target_shape)

    def _resolve(self, input_shape):
        n = 1
        for s in input_shape[1:]:
            n *= s
        known = 1
        for s in self.target_shape:
            if s != -1:
                known *= s
        shape = tuple(n // known if s == -1 else s for s in self.target_shape)
        total = 1
        for s in shape:
            total *= s
        if total != n or list(self.target_shape).count(-1) > 1:
            raise ValueError("total size of new array must be unchanged, input_shape = %s, output_shape = %s"
                             % (list(input_shape[1:]), list(self.target_shape)))
        return shape

    def call(self, inputs, **kwargs):
        return ops.reshape(inputs, (None,) + self._resolve(tuple(inputs.data.shape)))

    def compute_output_shape(self, input_shape):
        return (input_shape[0],) + self._resolve(tuple(input_shape))

    def get_config(self):
        c = Layer.get_config(self)
        c.update(target_shape=self.target_shape)
        return c


class Concatenate(Layer):
    def __init__(self, axis=-1, **kwargs):
        Layer.__init__(self, **kwargs)
        self.axis = axis

    def call(self, inputs, **kwargs):
        return ops.concat(inputs, self.axis)

    def compute_output_shape(self, input_shape):
        shapes = [list(s) for s in input_shape]
        ax = self.axis if self.axis >= 0 else len(shapes[0]) + self.axis
        out = list(shapes[0])
        out[ax] = sum(s[ax] for s in shapes)
        return tuple(out)

    def get_config(self):
        c = Layer.get_config(self)
        c.update(axis=self.axis)
        return c


class Add(Layer):
    def call(self, inputs, **kwargs):
        return ops.add_n(inputs)

    def compute_output_shape(self, input_shape):
        # Keras broadcasting: take the highest-rank / largest shape
        best = input_shape[0]
        for s in input_shape[1:]:
            if len(s) > len(best):
                best = s
        return tuple(best)


class Multiply(Layer):
    """tf.keras.layers.Multiply: the elementwise product of same-shaped inputs.  ONN's products (onn.py:94) are
    served by the planner's field-aware kernel; a product the planner did not claim runs here on b2ctr_ewise."""

    def compute_output_shape(self, input_shape):
        shapes = [tuple(s) for s in input_shape]
        if len(shapes) < 2:
            raise ValueError("A merge layer should be called on a list of at least 2 inputs. Got %d inputs."
                             % len(shapes))
        for s in shapes[1:]:
            if tuple(s[1:]) != tuple(shapes[0][1:]):
                raise ValueError("Multiply: operands of shapes %s and %s differ (embedding dimensions %s and %s)"
                                 % (shapes[0], s, shapes[0][-1], s[-1]))
        return shapes[0]

    def call(self, inputs, **kwargs):
        return ops.multiply(list(inputs))


def multiply(inputs, **kwargs):
    """The functional interface to Multiply (tf.keras.layers.multiply)."""
    return Multiply(**kwargs)(inputs)


class _ShapeProbe(object):
    """What Lambda.compute_output_shape hands its function to learn the output shape without running it: the
    backend functions (``deepctr_b200.backend``) map a probe to a probe of their result's shape."""

    def __init__(self, shape, summed_from=None):
        self.shape = tuple(shape)
        self.summed_from = summed_from      # (probe, axis) when this is backend.sum's result on ``probe``


class Lambda(Layer):
    """tf.keras.layers.Lambda.  ``function`` receives / returns Vars; only ``ops`` functions make
    sense inside (DenseFeat.transform_fn, deepctr/inputs.py:170)."""

    def __init__(self, function, output_shape=None, **kwargs):
        Layer.__init__(self, **kwargs)
        self.function = function
        self._out_shape = output_shape
        self.reduces_last_axis = False

    def call(self, inputs, **kwargs):
        return self.function(inputs)

    def compute_output_shape(self, input_shape):
        """``output_shape`` when given; over a list of inputs the shape of the highest-rank one (the broadcast result
        of an elementwise lambda such as ``x[0] * expand_dims(x[1], -1)``), so that the Lambda has one output."""
        if self._out_shape is not None:
            return self._out_shape
        if not isinstance(input_shape, list):
            x = _ShapeProbe(input_shape)
            try:
                probe = self.function(x)
            except Exception:
                probe = None
            if isinstance(probe, _ShapeProbe):       # e.g. ONN's Lambda(lambda x: K.sum(x, axis=-1))
                # the planner serves a sum over the last axis of the input from its own product kernel
                self.reduces_last_axis = (probe.summed_from is not None and probe.summed_from[0] is x
                                          and probe.summed_from[1] == len(x.shape) - 1)
                return probe.shape
        if isinstance(input_shape, list) and input_shape and isinstance(input_shape[0], (list, tuple)):
            return tuple(max(input_shape, key=len))
        return input_shape


# ================================================================================================
# Model
# ================================================================================================
class Optimizer(object):
    def __init__(self, name, lr):
        self.name, self.lr, self.iterations = name, lr, 0
        self.step_dev = None        # Adam: step count in device memory (advanced once per step, see begin_step)

    def begin_step(self):
        """Called once per training step before the first apply().  Adam keeps its step count on the device so
        that the whole step, optimizer included, is replayable as a CUDA graph."""
        if self.name == "adam":
            if self.step_dev is None:
                self.step_dev = torch.empty((1,), dtype=torch.int64, device=device())
                self.step_dev.copy_(torch.tensor([self.iterations - 1], dtype=torch.int64))
            K.counter_add(self.step_dev, 1)

    def apply_all(self, ws):
        """One optimizer step for a list of weights (SGD: a single multi-tensor launch)."""
        if self.name == "sgd":
            live = [w for w in ws if w.grad is not None]
            gs = [w.grad if w.grad.is_contiguous() else w.grad.contiguous() for w in live]
            if any(g.numel() != w.data.numel() for g, w in zip(gs, live)):
                raise ValueError("gradient / weight size mismatch")
            K.sgd_step_multi([w.data for w in live], gs, self.lr, [w.l2 for w in live])
            for w in live:
                w.grad = None
            return
        for w in ws:
            self.apply(w)

    def apply(self, w):
        g = w.grad
        if g is None:
            return
        if not g.is_contiguous():
            g = g.contiguous()
        if self.name == "sgd":
            K.sgd_step(w.data, g, self.lr, w.l2)
        elif self.name == "adam":
            st = w.opt_state
            if "m" not in st:
                st["m"] = torch.zeros_like(w.data)
                st["v"] = torch.zeros_like(w.data)
                K.fill(st["m"], 0.0)
                K.fill(st["v"], 0.0)
            if self.step_dev is not None:
                K.adam_step_dev(w.data, g, st["m"], st["v"], self.lr, self.step_dev, l2=w.l2)
            else:
                K.adam_step(w.data, g, st["m"], st["v"], self.lr, self.iterations, l2=w.l2)
        elif self.name == "adagrad":
            st = w.opt_state
            if "acc" not in st:
                st["acc"] = torch.empty_like(w.data)
                K.fill(st["acc"], 0.1)    # Keras initial_accumulator_value
            K.adagrad_step(w.data, g, st["acc"], self.lr, l2=w.l2)
        else:
            raise ValueError("unknown optimizer %r" % self.name)
        w.grad = None


def get_optimizer(opt):
    if isinstance(opt, Optimizer):
        return opt
    if isinstance(opt, str):
        o = opt.lower()
        defaults = {"sgd": 0.01, "adam": 1e-3, "adagrad": 1e-3}
        if o not in defaults:
            raise ValueError("unsupported optimizer %r (sgd, adam, adagrad)" % opt)
        return Optimizer(o, defaults[o])
    raise ValueError("optimizer must be a name or an Optimizer")


def SGD(learning_rate=0.01, **kw):
    return Optimizer("sgd", kw.get("lr", learning_rate))


def Adam(learning_rate=1e-3, **kw):
    return Optimizer("adam", kw.get("lr", learning_rate))


def Adagrad(learning_rate=1e-3, **kw):
    return Optimizer("adagrad", kw.get("lr", learning_rate))


def E_labels(t):
    return t


class History(object):
    def __init__(self):
        self.history = {}


class Model(object):
    """tf.keras.Model (functional).  compile / fit / predict / evaluate / train_on_batch /
    test_on_batch / get_weights / set_weights / save_weights / load_weights - what
    examples/run_classification_criteo.py:44-50 and tests/utils.py:366-378 use."""

    def __init__(self, inputs, outputs, name=None):
        self.inputs = _flatten(inputs)
        self.outputs = outputs if isinstance(outputs, KTensor) else _flatten(outputs)
        self.name = name or "model"
        self._order = self._toposort()
        self.layers = []
        seen = set()
        for node in self._order:
            if id(node.layer) not in seen:
                seen.add(id(node.layer))
                self.layers.append(node.layer)
        self.input_names = [t.name for t in self.inputs]
        self.optimizer = None
        self.loss = None
        self.metrics_names = ["loss"]
        self.stop_training = False
        from .inputs import EmbeddingPlanner
        self.planner = EmbeddingPlanner(self)
        self._feeder = None
        self.dist = None           # the process group's DistContext when compiled for multi-GPU training

    # ---- graph -----------------------------------------------------------------------------
    def _toposort(self):
        order, state = [], {}

        def visit(t):
            node = t.node
            if id(node) in state:
                return
            state[id(node)] = 1
            for i in _flatten(node.inputs):
                visit(i)
            order.append(node)

        for t in _flatten(self.outputs):
            visit(t)
        # inputs that no output depends on are still legal model inputs
        return order

    def get_layer(self, name):
        for l in self.layers:
            if l.name == name:
                return l
        raise ValueError("No such layer: %s" % name)

    @property
    def weights(self):
        ws, seen = [], set()
        for l in self.layers:
            for w in l.weights:
                if id(w) not in seen:
                    seen.add(id(w))
                    ws.append(w)
        return ws

    @property
    def trainable_weights(self):
        return [w for w in self.weights if w.trainable]

    def get_weights(self):
        return [w.value() for w in self.weights]

    def set_weights(self, values):
        ws = self.weights
        if len(ws) != len(values):
            raise ValueError("model has %d weights, got %d arrays" % (len(ws), len(values)))
        for w, v in zip(ws, values):
            w.set_value(v)

    def save_weights(self, path):
        """h5py is not available in this image: weights are stored as .npz keyed by weight name
        (the reference's h5 layout is SURVEY.md section 8f row n1)."""
        np.savez(path if str(path).endswith(".npz") else str(path) + ".npz",
                 **{w.name: w.value() for w in self.weights})

    def load_weights(self, path):
        """By name; a checkpoint of an identically BUILT model whose automatic layer names differ (a second
        model of the same process: ``dnn_1`` vs ``dnn``) is matched by topology order + shapes, like Keras' h5
        loader does."""
        p = path if str(path).endswith(".npz") else str(path) + ".npz"
        data = np.load(p)
        ws = self.weights
        if all(w.name in data for w in ws):
            for w in ws:
                w.set_value(data[w.name])
            return
        keys = list(data.files)                  # np.savez keeps insertion (= topology) order
        if len(keys) != len(ws):
            missing = [w.name for w in ws if w.name not in data]
            raise ValueError("weight %s missing from %s (and %d stored arrays cannot be matched to %d weights by "
                             "order)" % (missing[0], p, len(keys), len(ws)))
        for w, k in zip(ws, keys):
            if tuple(data[k].shape) != tuple(w.shape):
                raise ValueError("weight %s missing from %s; by order it would take %s of shape %s, expected %s"
                                 % (w.name, p, k, data[k].shape, w.shape))
        for w, k in zip(ws, keys):
            w.set_value(data[k])

    def count_params(self):
        return sum(w.numel() for w in self.weights)

    def summary(self, print_fn=print):
        print_fn("Model: %s" % self.name)
        for l in self.layers:
            print_fn("  %-40s %-28s params=%d" % (l.name, l.__class__.__name__,
                                                  sum(w.numel() for w in l._weights)))
        print_fn("Total params: %d" % self.count_params())

    # ---- execution ---------------------------------------------------------------------------
    def compile(self, optimizer="adam", loss=None, metrics=None, embedding_update="auto", distributed="auto",
                step_graph="auto", **kw):
        """``embedding_update``: 'dense' = Keras semantics (dense gradient + dense optimizer + l2 on
        the whole table, SURVEY.md App. C; O(vocab) per step), 'sparse' = fused row-wise SGD scatter
        (O(batch); l2 on tables must be 0), 'auto' = dense below 4M table elements."""
        self.optimizer = get_optimizer(optimizer)
        self.loss = loss
        known = ("binary_crossentropy", "bce", "mse", "mean_squared_error", "logloss")
        extra = [m for m in (metrics or []) if not (isinstance(m, str) and m in known)]
        if extra:
            import warnings
            warnings.warn("metrics %r are not computed by this runtime (fit reports loss / val_loss only)" % (extra,))
        self.metrics = metrics or []
        self.metrics_names = ["loss"] + [m if isinstance(m, str) else m.__name__ for m in self.metrics]
        if embedding_update not in ("auto", "dense", "sparse", "sparse_deterministic"):
            raise ValueError("embedding_update must be auto / dense / sparse / sparse_deterministic")
        self.planner.configure(self.optimizer, embedding_update)
        # CUDA-graph replay of the training step ('auto': on whenever the step is capturable)
        from . import ops as _ops
        self.step_graph = step_graph if os.environ.get("B2CTR_STEP_GRAPH", "1") != "0" else "off"
        self._step_graphs, self._graph_pool, self._eager_steps, self._eager_shapes = {}, None, 0, {}
        self.replayed_launches = 0             # kernels executed through graph replays (bench accounting)
        self._uncapturable0 = _ops.UNCAPTURABLE
        # multi-GPU (one process per GPU): dense weights data-parallel, fast-path tables row-sharded
        self.dist = None
        if distributed not in (None, False):
            import torch.distributed as tdist
            if tdist.is_available() and tdist.is_initialized() and tdist.get_world_size() > 1:
                from . import parallel
                self.dist = parallel.DistContext()
                self.planner.set_dist(self.dist)

    def _materialize(self):
        for w in self.weights:
            w.materialize()

    def _check_ids(self):
        """Raise like TF-CPU's Embedding does (InvalidArgument: indices[...] is not in [0, V)) when a gather
        kernel met an id outside its table since the last check.  The kernels themselves stay memory-safe:
        such ids read a zero row and are never written (deepctr/inputs.py:101-130 relies on Keras for this).
        Called where the host synchronises anyway (end of predict / evaluate / fit epoch, train_on_batch)."""
        n = K.embed_oob_count(reset=True)
        if n:
            raise ValueError("%d embedding lookups used an id outside [0, vocabulary_size): check the "
                             "vocabulary_size of the feature columns against the data (unseen categories at "
                             "predict time, -1 for missing values...); the rows were read as zeros" % n)

    def close(self):
        """Release what must not outlive the process group: captured step graphs (they hold NCCL kernels) and
        the CUDA-IPC mappings of the other ranks' table shards.  Call before dist.destroy_process_group()."""
        self._step_graphs = {}
        self._graph_pool = None
        if self.planner.peers is not None:
            for pt in self.planner.peers[:2]:
                if pt is not None:
                    pt.close()
            self.planner.peers = None
        gc.collect()
        if torch.cuda.is_available():
            torch.cuda.synchronize()
            torch.cuda.ipc_collect()

    def _run(self, feed, training, upto=None):
        """Execute the graph; returns {id(KTensor): Var}.  ``upto``: stop before this node."""
        values = {}
        for t in self.inputs:
            values[id(t)] = feed[t.name]
        self.planner.begin_step(feed, training)
        for node in self._order:
            if isinstance(node.layer, InputLayer):
                t = node.outputs[0]
                if id(t) not in values:
                    raise ValueError("missing model input %r" % t.name)
                continue
            if node is upto:
                break
            launch = self.planner.launches.get(id(node))
            if launch is not None:        # a planned node, or a fused chain's first node that serves the later nodes
                self.planner.results.update(launch(values, training))
            # popped: what a step's launches made is held by that step's values and tape only
            planned = self.planner.results.pop(id(node), None)
            if planned is not None:       # served by the planner (inputs.EmbeddingPlanner), with the result's own mask
                values[id(node.outputs[0])] = planned
                continue
            ins = _map_structure(lambda t: values[id(t)], node.inputs)
            out = node.layer._invoke(ins, training)
            outs = _flatten(out) if len(node.outputs) > 1 else [out]
            for t, v in zip(node.outputs, outs):
                values[id(t)] = v
        return values

    def _feed(self, x, batch_slice=None):
        from .inputs import Feeder
        if self._feeder is None:
            self._feeder = Feeder(self)
        return self._feeder.feed(x, batch_slice)

    def _head(self):
        """(logit KTensor, PredictionLayer node) when the output is produced by a PredictionLayer -
        lets prediction + loss + gradient run as ONE kernel (b2ctr_predict_loss)."""
        from .layers.core import PredictionLayer
        out = self.outputs if isinstance(self.outputs, KTensor) else self.outputs[0]
        node = out.node
        if isinstance(node.layer, PredictionLayer) and isinstance(node.inputs, KTensor):
            return node.inputs, node
        return None, None

    def _task_for_loss(self):
        loss = self.loss
        if loss in ("binary_crossentropy", "bce"):
            return L.TASK_BINARY
        if loss in ("mse", "mean_squared_error"):
            return L.TASK_REGRESSION
        raise ValueError("unsupported loss %r (binary_crossentropy, mse)" % (loss,))

    def predict_on_batch(self, x):
        self._materialize()
        feed = self._feed(x)
        vals = self._run(feed, False)
        out = self.outputs if isinstance(self.outputs, KTensor) else self.outputs[0]
        return contiguous(vals[id(out)]).reshape(-1, 1)

    def _stage_batch(self, x, y, stream=None):
        """Pack + H2D one batch (optionally on a side stream); returns (feed, labels, ready event, slot)."""
        if stream is None:
            feed = self._feed(x)
            return feed, self._feeder.labels(y), None, self._feeder.slot
        with torch.cuda.stream(stream):
            feed = self._feed(x)
            labels = self._feeder.labels(y)
            ev = torch.cuda.Event()
            ev.record(stream)
        return feed, labels, ev, self._feeder.slot

    def _loss_step(self, x, y, train, staged=None):
        """forward (+ backward + update when ``train``); returns the device loss_sum tensor [1], the
        predictions and the batch size - no host synchronisation here.

        Training steps are replayed as CUDA graphs once warm: the whole step (fused gather, GEMMs, loss,
        backward, scatter/optimizer kernels) is captured per staging-ring slot, so a step costs one
        cudaGraphLaunch on the host instead of ~70 kernel launches."""
        if self.optimizer is None:
            raise RuntimeError("You must compile your model before training/testing.")
        self._materialize()
        if staged is None:
            staged = self._stage_batch(x, y)
        feed, labels, ev, slot = staged
        if ev is not None:
            torch.cuda.current_stream().wait_event(ev)
        try:
            if train and self._graph_eligible():
                key = self._graph_key(feed, labels)
                ent = self._step_graphs.get(key)
                shapes = tuple(it[2] for it in key[0])
                if (ent is None and self._eager_steps >= 2 and self._eager_shapes.get(shapes, 0) >= 1
                        and len(self._step_graphs) < 8):
                    # (a batch shape is captured only after it ran eagerly once: first-use work - per-shape launch
                    # plans, lazily created state - includes host-synchronous copies that a capture cannot hold)
                    ent = self._capture_step(key, feed, labels)
                if ent is not None:
                    self.optimizer.iterations += 1
                    ent[0].replay()
                    self.replayed_launches += ent[4]
                    return ent[1], ent[2], ent[3]
            out = self._loss_step_impl(feed, labels, train)
            if train:
                self._eager_steps += 1
                shapes = tuple(tuple(v.data.shape) if isinstance(v, Var) else tuple(v.shape)
                               for _, v in sorted(feed.items()) if (v.data if isinstance(v, Var) else v) is not None)
                self._eager_shapes[shapes] = self._eager_shapes.get(shapes, 0) + 1
            return out
        finally:
            self._feeder.consumed(slot)

    # ---- CUDA-graph replay of the training step ---------------------------------------------------
    def _graph_eligible(self):
        from . import ops
        if self.step_graph in (False, None, "off") or K.PROFILE is not None:
            return False
        if self.dist is not None and self.planner.sharded and not self.planner.peer_mode:
            return False                       # NCCL all-to-all transport: split sizes are read on the host
        return ops.UNCAPTURABLE == self._uncapturable0

    def _graph_key(self, feed, labels):
        items = []
        for name in sorted(feed):
            v = feed[name]
            t = v.data if isinstance(v, Var) else v
            if t is not None:
                items.append((name, t.data_ptr(), tuple(t.shape), tuple(t.stride()), str(t.dtype)))
        return (tuple(items), labels.data_ptr(), tuple(labels.shape), float(self.optimizer.lr),
                torch.cuda.current_device())

    def _capture_step(self, key, feed, labels):
        from . import ops
        it0 = self.optimizer.iterations
        n0 = L.launch_count()
        graph = torch.cuda.CUDAGraph()
        # No garbage collection while the stream captures: a collection can run the destructors of unrelated dead
        # CUDA objects (graphs, pinned host buffers, events), and some of them make CUDA calls a capture forbids.
        gc_enabled = gc.isenabled()
        gc.disable()
        try:
            with torch.cuda.graph(graph, pool=self._graph_pool, capture_error_mode="thread_local"):
                loss_sum, pred, batch = self._loss_step_impl(feed, labels, True)
        except Exception as exc:               # something on this model's path cannot be captured: stay eager
            import traceback
            import warnings
            where = "".join(traceback.format_tb(exc.__traceback__)[-4:])
            warnings.warn("step graph capture failed (%s: %s); training continues with eager launches\n%s"
                          % (type(exc).__name__, exc, where))
            self.step_graph = "off"
            self.optimizer.iterations = it0
            for w in self.weights:             # nothing ran on the device; drop the half-built python state
                w.grad = None
            return None
        finally:
            if gc_enabled:
                gc.enable()
        self.optimizer.iterations = it0        # capturing does not execute the step
        if ops.UNCAPTURABLE != self._uncapturable0:
            self.step_graph = "off"
            return None
        if self._graph_pool is None:
            self._graph_pool = graph.pool()
        ent = (graph, loss_sum, pred, batch, L.launch_count() - n0)
        self._step_graphs[key] = ent
        return ent

    def _loss_step_impl(self, feed, labels, train):
        logit_t, head = self._head()
        if head is None:
            raise ValueError("training needs a PredictionLayer output (all builders end with one)")
        player = head.layer
        task = self._task_for_loss()
        if (task == L.TASK_BINARY) != (player.task == "binary"):
            raise ValueError("loss %r does not match PredictionLayer(task=%r)" % (self.loss, player.task))
        tape = Tape() if train else None
        with recording(tape):
            vals = self._run(feed, train, upto=head)
            logit = vals[id(logit_t)]
            lt = contiguous(logit).reshape(-1)
            bias = player.global_bias.materialize() if player.use_bias else None
            pred, dlogit, dbias, loss_sum = K.predict_loss(lt, bias, labels, task, want_grad=train)
        if train:
            logit.requires_grad = True
            add_grad(logit, dlogit.reshape(logit.data.shape))
            if bias is not None:
                player.global_bias.grad = dbias
            self.optimizer.iterations += 1
            tape.ctx["optimizer"] = self.optimizer
            tape.backward()
            dense = [w for w in self.trainable_weights if not w.sparse_grad]
            if self.dist is not None:
                from . import parallel
                parallel.reduce_dense_grads(
                    self.dist, dense,
                    lambda src, flat, off: K.copy2d(src.reshape(1, -1), src.numel(), flat, flat.numel(), 1,
                                                    src.numel(), dst_off=off),
                    lambda flat, f: K.add_n([flat], scales=[f], out=flat))
            self.optimizer.begin_step()
            self.optimizer.apply_all(dense)
        return loss_sum, pred, lt.shape[0]

    def train_step(self, x, y):
        """One optimisation step without any host synchronisation: returns the device tensor [1]
        holding the batch's summed loss (train_on_batch = this + .item() / batch)."""
        return self._loss_step(x, y, True)[0]

    def train_on_batch(self, x, y, **kw):
        loss_sum, _, batch = self._loss_step(x, y, True)
        loss = float(loss_sum.item()) / batch + self._reg_loss()
        self._check_ids()
        return loss

    def test_on_batch(self, x, y, **kw):
        loss_sum, _, batch = self._loss_step(x, y, False)
        loss = float(loss_sum.item()) / batch + self._reg_loss()
        self._check_ids()
        return loss

    def _reg_loss(self):
        tot = 0.0
        for w in self.weights:
            if w.l2 > 0 and w.data is not None and w.numel() <= (1 << 22):
                tot += w.l2 * float((w.value().astype(np.float64) ** 2).sum())
        return tot

    @staticmethod
    def _num_samples(x):
        if isinstance(x, dict):
            x = list(x.values())
        first = x[0] if isinstance(x, (list, tuple)) else x
        return len(first)

    def predict(self, x, batch_size=32, verbose=0, **kw):
        n = self._num_samples(x)
        from .inputs import slice_inputs
        outs = []
        for s in range(0, n, batch_size):
            outs.append(self.predict_on_batch(slice_inputs(x, slice(s, min(n, s + batch_size)))).cpu())
        if outs:
            self._check_ids()
        return torch.cat(outs, 0).numpy() if outs else np.zeros((0, 1), np.float32)

    def evaluate(self, x, y, batch_size=32, verbose=0, **kw):
        from .inputs import slice_inputs
        n = self._num_samples(x)
        y = np.asarray(y)
        tot = 0.0
        for s in range(0, n, batch_size):
            sl = slice(s, min(n, s + batch_size))
            ls, _, b = self._loss_step(slice_inputs(x, sl), y[sl], False)
            tot += float(ls.item())
        if n:
            self._check_ids()
        return tot / max(n, 1) + self._reg_loss()

    def fit(self, x=None, y=None, batch_size=32, epochs=1, verbose=1, validation_split=0.0,
            validation_data=None, shuffle=True, callbacks=None, **kw):
        from .inputs import slice_inputs
        if callbacks:
            import warnings
            warnings.warn("fit(callbacks=...) is not supported by this runtime: %d callback(s) ignored" % len(callbacks))
        n = self._num_samples(x)
        y = np.asarray(y)
        hist = History()
        val = None
        if validation_data is not None:
            val = validation_data
        elif validation_split and 0.0 < validation_split < 1.0:
            split = int(n * (1.0 - validation_split))      # Keras: the LAST fraction, before shuffling
            val = (slice_inputs(x, slice(split, n)), y[split:])
            x, y, n = slice_inputs(x, slice(0, split)), y[:split], split
        rng = np.random.RandomState(kw.get("seed", None)) if shuffle else None
        for ep in range(epochs):
            perm = rng.permutation(n) if shuffle else None
            cnt = 0
            nsteps = (n + batch_size - 1) // batch_size
            # every step's loss is read back (4 B, asynchronous D2H into pinned memory); the host only
            # waits at the end of the epoch, so staging batch i+1 overlaps the kernels of batch i
            host_losses = getattr(self, "_host_losses", None)
            if host_losses is None or host_losses.numel() < nsteps:
                host_losses = torch.empty((max(nsteps, 64),), dtype=torch.float32)
                try:
                    host_losses = host_losses.pin_memory()
                except Exception:
                    pass
                self._host_losses = host_losses
            # Input pipeline: a producer thread packs batch after batch into the staging ring (native
            # thread-pool memcpy into pinned memory + H2D on a side stream) and runs AHEAD of this thread by up
            # to RING-1 batches; this thread only replays the step graph per staged batch.  The semaphore
            # counts launched steps: ring slot (j mod RING) is refilled only after step j-RING was enqueued
            # (its `consumed` event then orders the H2D after the kernels that read the slot).
            import queue
            import sys
            import threading
            from .inputs import Feeder
            if not hasattr(self, "_stage_stream"):
                self._stage_stream = torch.cuda.Stream()
            starts = list(range(0, n, batch_size))

            def batch_of(s):
                idx = perm[s:s + batch_size] if perm is not None else slice(s, min(n, s + batch_size))
                return slice_inputs(x, idx), y[idx]

            self._materialize()
            if self._feeder is None:
                self._feeder = Feeder(self)
            dev_index = torch.cuda.current_device()
            staged_q = queue.Queue()
            # the first batch is staged right here: the first step is on the device before the producer thread
            # has even started (thread start + first wake-up cost ~0.5 ms of an otherwise idle GPU per epoch)
            first = None
            if starts:
                bx0, by0 = batch_of(starts[0])
                first = self._stage_batch(bx0, by0, self._stage_stream)
            permits = threading.Semaphore(Feeder._RING - 2)
            stop = [False]

            def producer():
                try:
                    torch.cuda.set_device(dev_index)
                    for s in starts[1:]:
                        permits.acquire()
                        if stop[0]:
                            return
                        bx, by = batch_of(s)
                        staged_q.put(self._stage_batch(bx, by, self._stage_stream))
                except BaseException as exc:       # surfaced by the consumer loop
                    staged_q.put(exc)

            worker = threading.Thread(target=producer, name="b2ctr-staging", daemon=True)
            # the producer spends most of its time in GIL-releasing copies; a short switch interval keeps its
            # Python stretches from holding the interpreter while this thread needs ~0.1 ms per step
            switch0 = sys.getswitchinterval()
            sys.setswitchinterval(1e-4)
            worker.start()
            try:
                for i, s in enumerate(starts):
                    staged = first if i == 0 else staged_q.get()
                    if isinstance(staged, BaseException):
                        raise staged
                    ls, _, b = self._loss_step(None, None, True, staged=staged)
                    permits.release()
                    # (graph replay: `ls` is the graph's static output; the copy below is stream-ordered
                    # before the next replay overwrites it)
                    host_losses[i:i + 1].copy_(ls, non_blocking=True)
                    cnt += b
                torch.cuda.synchronize()
            finally:
                stop[0] = True
                permits.release()
                worker.join()
                sys.setswitchinterval(switch0)
            self.d2h_bytes = getattr(self, "d2h_bytes", 0) + 4 * nsteps + 8
            self._check_ids()
            tot = float(host_losses[:nsteps].double().sum()) if nsteps else 0.0
            logs = {"loss": tot / max(cnt, 1) + self._reg_loss()}
            if val is not None:
                logs["val_loss"] = self.evaluate(val[0], val[1], batch_size=batch_size)
            for k, v in logs.items():
                hist.history.setdefault(k, []).append(v)
            if verbose:
                print("Epoch %d/%d - %s" % (ep + 1, epochs,
                                            " - ".join("%s: %.4f" % kv for kv in logs.items())))
        return hist
