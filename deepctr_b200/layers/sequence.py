"""Host mirror of deepctr/layers/sequence.py for the hot path: SequencePoolingLayer (:41-120),
WeightedSequenceLayer (:123-197), AttentionSequencePoolingLayer (:200-315), Transformer (:431-651),
PositionEncoding (:654-703) and KMaxPooling (:818-874).

When these layers hang directly off an embedding lookup of a model input (the shape
``get_varlen_pooling_list`` produces) the EmbeddingPlanner folds them into the fused gather and their
``call`` never runs; the standalone kernels below serve every other use."""
import numpy as np

from .. import engine as E
from .. import kernels as K
from .. import ops
from ..engine import Layer, Constant, TruncatedNormal, glorot_uniform
from .core import LocalActivationUnit
from .normalization import Dropout, LayerNormalization

# limits of the fused attention kernel (b2ctr_mha_fwd / _bwd)
MHA_MAX_T = 128
MHA_MAX_HEAD = 64


class SequencePoolingLayer(Layer):
    """sum / mean / max over the valid positions of [B,T,E] -> [B,1,E]."""

    def __init__(self, mode='mean', supports_masking=False, **kwargs):
        if mode not in ['sum', 'mean', 'max']:
            raise ValueError("mode must be sum or mean")
        self.mode = mode
        self.eps = 1e-8
        Layer.__init__(self, **kwargs)
        self.supports_masking = supports_masking

    def build(self, input_shape):
        if not self.supports_masking:
            self.seq_len_max = int(input_shape[0][1])
        self.built = True

    def call(self, seq_value_len_list, mask=None, **kwargs):
        if self.supports_masking:
            if mask is None:
                raise ValueError("When supports_masking=True,input must support masking")
            seq = seq_value_len_list
            m = mask.materialize()
            return ops.seqpool(seq, self.mode, mask_u8=m)
        seq, lengths = seq_value_len_list
        return ops.seqpool(seq, self.mode, lengths=lengths)

    def compute_output_shape(self, input_shape):
        if self.supports_masking:
            return (None, 1, input_shape[-1])
        return (None, 1, input_shape[0][-1])

    def compute_mask(self, inputs, mask=None):
        return None

    def get_config(self):
        config = {'mode': self.mode, 'supports_masking': self.supports_masking}
        base = Layer.get_config(self)
        return dict(list(base.items()) + list(config.items()))


class WeightedSequenceLayer(Layer):
    """[B,T,E] * (masked, optionally soft-maxed) per-position weights [B,T,1] -> [B,T,E]."""

    def __init__(self, weight_normalization=True, supports_masking=False, **kwargs):
        Layer.__init__(self, **kwargs)
        self.weight_normalization = weight_normalization
        self.supports_masking = supports_masking

    def build(self, input_shape):
        if not self.supports_masking:
            self.seq_len_max = int(input_shape[0][1])
        self.built = True

    def call(self, input_list, mask=None, **kwargs):
        if self.supports_masking:
            if mask is None:
                raise ValueError("When supports_masking=True,input must support masking")
            key_input, value_input = input_list
            m = mask[0].materialize()
            return ops.weighted_seq(key_input, value_input, self.weight_normalization, mask_u8=m)
        key_input, key_length_input, value_input = input_list
        return ops.weighted_seq(key_input, value_input, self.weight_normalization, lengths=key_length_input)

    def compute_output_shape(self, input_shape):
        return input_shape[0]

    def compute_mask(self, inputs, mask=None):
        if self.supports_masking:
            return mask[0] if mask is not None else None
        return None

    def get_config(self):
        config = {'weight_normalization': self.weight_normalization, 'supports_masking': self.supports_masking}
        base = Layer.get_config(self)
        return dict(list(base.items()) + list(config.items()))


class AttentionSequencePoolingLayer(Layer):
    """DIN attentional pooling, deepctr/layers/sequence.py:200-315.
    score = LocalActivationUnit([q, keys]); masked fill (0, or -2^32+1 then softmax when
    weight_normalization); out = score @ keys -> [B,1,E] (or the scores when return_score)."""

    def __init__(self, att_hidden_units=(80, 40), att_activation='sigmoid', weight_normalization=False,
                 return_score=False, supports_masking=False, **kwargs):
        self.att_hidden_units = att_hidden_units
        self.att_activation = att_activation
        self.weight_normalization = weight_normalization
        self.return_score = return_score
        Layer.__init__(self, **kwargs)
        self.supports_masking = supports_masking

    def build(self, input_shape):
        if not self.supports_masking:
            if not isinstance(input_shape, list) or len(input_shape) != 3:
                raise ValueError('A `AttentionSequencePoolingLayer` layer should be called '
                                 'on a list of 3 inputs')
            if len(input_shape[0]) != 3 or len(input_shape[1]) != 3 or len(input_shape[2]) != 2:
                raise ValueError(
                    "Unexpected inputs dimensions,the 3 tensor dimensions are %d,%d and %d , expect to be 3,3 and 2" % (
                        len(input_shape[0]), len(input_shape[1]), len(input_shape[2])))
            if input_shape[0][-1] != input_shape[1][-1] or input_shape[0][1] != 1 or input_shape[2][1] != 1:
                raise ValueError('A `AttentionSequencePoolingLayer` layer requires '
                                 'inputs of a 3 tensor with shape (None,1,embedding_size),(None,T,embedding_size) and (None,1)'
                                 'Got different shapes: %s' % (input_shape))
        self.local_att = self._track(LocalActivationUnit(
            self.att_hidden_units, self.att_activation, l2_reg=0, dropout_rate=0, use_bn=False, seed=1024,
            name=self.name + "/local_activation_unit"))
        self.local_att._maybe_build([tuple(input_shape[0]), tuple(input_shape[1])])
        self.built = True

    def call(self, inputs, mask=None, training=None, **kwargs):
        if self.supports_masking:
            if mask is None:
                raise ValueError("When supports_masking=True,input must support masking")
            queries, keys = inputs
            km = mask[-1]
            if km is None:
                raise ValueError("When supports_masking=True,input must support masking")
            key_mask = km.materialize()
        else:
            queries, keys, keys_length = inputs
            key_mask = E.KMask(lengths=keys_length.data.reshape(-1), maxlen=keys.data.shape[1]).materialize()
        from .. import kernels as K
        with K.profile_tag("din_att"):
            score = self.local_att.call([queries, keys], training=training)      # [B,T,1]
            return ops.din_attention_pool(score, keys, key_mask, self.weight_normalization, self.return_score)

    def compute_output_shape(self, input_shape):
        if self.return_score:
            return (None, 1, input_shape[1][1])
        return (None, 1, input_shape[0][-1])

    def compute_mask(self, inputs, mask=None):
        return None

    def get_config(self):
        config = {'att_hidden_units': self.att_hidden_units, 'att_activation': self.att_activation,
                  'weight_normalization': self.weight_normalization, 'return_score': self.return_score,
                  'supports_masking': self.supports_masking}
        base = Layer.get_config(self)
        return dict(list(base.items()) + list(config.items()))


class Transformer(Layer):
    """Simplified Transformer (Vaswani et al. 2017) of the reference, deepctr/layers/sequence.py:431-651.

    Q / K / V and the feed-forward ``relu(x fw1) fw2`` run on the dense GEMMs; the masked multi-head attention
    (scores, key mask, blinding, softmax, query mask, dropout, weighted sum and the residual) is one fused kernel
    that keeps no [B, heads, T, T] tensor.  As in the reference, one LayerNormalization (``self.ln``) and one
    Dropout (``self.dropout``) serve both sites, and the queries and keys get separate PositionEncoding tables.
    Only ``attention_type='scaled_dot_product'`` is implemented."""

    def __init__(self, att_embedding_size=1, head_num=8, dropout_rate=0.0, use_positional_encoding=True, use_res=True,
                 use_feed_forward=True, use_layer_norm=False, blinding=True, seed=1024, supports_masking=False,
                 attention_type="scaled_dot_product", output_type="mean", **kwargs):
        if head_num <= 0:
            raise ValueError('head_num must be a int > 0')
        self.att_embedding_size = att_embedding_size
        self.head_num = head_num
        self.num_units = att_embedding_size * head_num
        self.use_res = use_res
        self.use_feed_forward = use_feed_forward
        self.seed = seed
        self.use_positional_encoding = use_positional_encoding
        self.dropout_rate = dropout_rate
        self.use_layer_norm = use_layer_norm
        self.blinding = blinding
        self.attention_type = attention_type
        self.output_type = output_type
        Layer.__init__(self, **kwargs)
        self.supports_masking = supports_masking

    def build(self, input_shape):
        embedding_size = int(input_shape[0][-1])
        if self.num_units != embedding_size:
            raise ValueError(
                "att_embedding_size * head_num must equal the last dimension size of inputs,got %d * %d != %d" % (
                    self.att_embedding_size, self.head_num, embedding_size))
        if self.attention_type in ("cos", "ln", "additive"):
            raise NotImplementedError("Transformer attention_type=%r is not implemented (only 'scaled_dot_product')"
                                      % (self.attention_type,))
        if self.attention_type != "scaled_dot_product":
            raise ValueError("attention_type must be [scaled_dot_product,cos,ln,additive]")
        self.seq_len_max = int(input_shape[0][-2])
        if tuple(input_shape[1][-2:]) != tuple(input_shape[0][-2:]):
            # the reference's key mask (sequence.py:581-591) only lines up with keys of the queries' shape
            raise ValueError("Transformer: queries and keys must have the same shape (T, E), got %s and %s"
                             % (tuple(input_shape[0][1:]), tuple(input_shape[1][1:])))
        if not (1 <= self.seq_len_max <= MHA_MAX_T and 1 <= self.att_embedding_size <= MHA_MAX_HEAD):
            raise ValueError("Transformer supports 1 <= T <= %d and 1 <= att_embedding_size <= %d, got T=%d, "
                             "att_embedding_size=%d" % (MHA_MAX_T, MHA_MAX_HEAD, self.seq_len_max,
                                                        self.att_embedding_size))
        self.W_Query = self.add_weight(name='query', shape=[embedding_size, self.num_units],
                                       initializer=TruncatedNormal(seed=self.seed))
        self.W_key = self.add_weight(name='key', shape=[embedding_size, self.num_units],
                                     initializer=TruncatedNormal(seed=self.seed + 1))
        self.W_Value = self.add_weight(name='value', shape=[embedding_size, self.num_units],
                                       initializer=TruncatedNormal(seed=self.seed + 2))
        if self.use_feed_forward:
            self.fw1 = self.add_weight('fw1', shape=[self.num_units, 4 * self.num_units],
                                       initializer=glorot_uniform(seed=self.seed))
            self.fw2 = self.add_weight('fw2', shape=[4 * self.num_units, self.num_units],
                                       initializer=glorot_uniform(seed=self.seed))
        # the reference creates these layers here: they take the next `dropout`, `layer_normalization` and
        # `position_encoding` names
        self.dropout = self._track(Dropout(self.dropout_rate, seed=self.seed, name=self.name + "/dropout"))
        self.ln = self._track(LayerNormalization(name=self.name + "/ln"))
        if self.use_layer_norm:         # Keras builds (and gives weights to) a layer when it is first called
            self.ln._maybe_build(tuple(input_shape[0]))
        if self.use_positional_encoding:
            self.query_pe = self._track(PositionEncoding(name=self.name + "/query_pe"))
            self.key_pe = self._track(PositionEncoding(name=self.name + "/key_pe"))
            self.query_pe._maybe_build(tuple(input_shape[0]))
            self.key_pe._maybe_build(tuple(input_shape[1]))
        self.built = True

    def call(self, inputs, mask=None, training=None, **kwargs):
        if self.supports_masking:
            if mask is None or mask[0] is None or mask[1] is None:
                raise ValueError("When supports_masking=True,input must support masking")
            queries, keys = inputs
            valid = dict(qmask=mask[0].materialize(), kmask=mask[1].materialize())
        else:
            queries, keys, query_len, key_len = inputs
            valid = dict(qlen=query_len, klen=key_len)
        if self.use_positional_encoding:
            queries = self.query_pe.call(queries)
            keys = self.key_pe.call(keys)
        q = ops.dense(queries, self.W_Query)
        k = ops.dense(keys, self.W_key)
        v = ops.dense(keys, self.W_Value)
        rate = self.dropout_rate if (training and self.dropout_rate) else 0.0
        seed = self.dropout.next_seed() if rate else 0
        scale = float(np.float32(1.0) / np.sqrt(np.float32(self.att_embedding_size)))
        result = ops.mha(q, k, v, self.head_num, scale, blinding=self.blinding, rate=rate, seed=seed,
                         res=queries if self.use_res else None, **valid)
        if self.use_layer_norm:
            result = self.ln.call(result)
        if self.use_feed_forward and self.use_res:
            hidden = ops.dense(result, self.fw1, activation="relu")
            hidden = self.dropout.call(hidden, training=training)
            fw2 = ops.dense(hidden, self.fw2)
            result = self.ln.call(result, residual=fw2) if self.use_layer_norm else ops.add(result, fw2)
        elif self.use_feed_forward and self.use_layer_norm:
            # without the residual the reference computes fw2, drops it and normalises the result a second time
            result = self.ln.call(result)
        if self.output_type in ("mean", "sum"):
            B, T, _ = result.shape
            return ops.seqpool(result, self.output_type, lengths=ops.full_lengths(B, T, result.data.device))
        return result

    def compute_output_shape(self, input_shape):
        if self.output_type in ("mean", "sum"):
            return (None, 1, self.num_units)
        return tuple(input_shape[0][:-1]) + (self.num_units,)

    def compute_mask(self, inputs, mask=None):
        return None

    def get_config(self):
        config = {'att_embedding_size': self.att_embedding_size, 'head_num': self.head_num,
                  'dropout_rate': self.dropout_rate, 'use_res': self.use_res,
                  'use_positional_encoding': self.use_positional_encoding, 'use_feed_forward': self.use_feed_forward,
                  'use_layer_norm': self.use_layer_norm, 'seed': self.seed, 'supports_masking': self.supports_masking,
                  'blinding': self.blinding, 'attention_type': self.attention_type, 'output_type': self.output_type}
        base = Layer.get_config(self)
        return dict(list(base.items()) + list(config.items()))


def sinusoid_table(T, num_units, zero_pad=False):
    """The initial PositionEncoding table (deepctr/layers/sequence.py:667-675): sin on even, cos on odd columns."""
    enc = np.array([[pos / np.power(10000, 2. * (i // 2) / num_units) for i in range(num_units)]
                    for pos in range(T)])
    enc[:, 0::2] = np.sin(enc[:, 0::2])
    enc[:, 1::2] = np.cos(enc[:, 1::2])
    if zero_pad:
        enc[0, :] = np.zeros(num_units)
    return enc


class PositionEncoding(Layer):
    """x + sqrt(E) * P[t] (deepctr/layers/sequence.py:654-703) as a bias over the per-sample [T*E] view: the
    forward is a rank-1 update, the table's gradient a column sum (ops.add_bias)."""

    def __init__(self, pos_embedding_trainable=True, zero_pad=False, scale=True, **kwargs):
        self.pos_embedding_trainable = pos_embedding_trainable
        self.zero_pad = zero_pad
        self.scale = scale
        Layer.__init__(self, **kwargs)

    def build(self, input_shape):
        _, T, num_units = input_shape
        self.lookup_table = self.add_weight("lookup_table", (T, num_units),
                                            initializer=Constant(sinusoid_table(T, num_units, self.zero_pad)),
                                            trainable=self.pos_embedding_trainable)
        self.built = True

    def call(self, inputs, mask=None, **kwargs):
        num_units = inputs.shape[-1]
        return ops.add_bias(inputs, self.lookup_table, scale=num_units ** 0.5 if self.scale else 1.0,
                            per_sample=True)

    def compute_output_shape(self, input_shape):
        return input_shape

    def compute_mask(self, inputs, mask=None):
        return mask

    def get_config(self):
        config = {'pos_embedding_trainable': self.pos_embedding_trainable, 'zero_pad': self.zero_pad,
                  'scale': self.scale}
        base = Layer.get_config(self)
        return dict(list(base.items()) + list(config.items()))


class KMaxPooling(Layer):
    """The k largest values along ``axis`` in descending order (tf.nn.top_k(sorted=True): equal values keep the
    lower index first), deepctr/layers/sequence.py:818-874.  An n-D input is viewed as [outer, n, inner] with n the
    pooled axis; the layer is one k-max stage of b2ctr_conv_stack over its inner columns, and in CCPM the planner
    (inputs.ConvStackPlan) runs it inside the launch of the whole convolution stack.  The gradient goes to the
    selected elements only.

    Deviation: ``axis == len(input_shape)`` passes the reference's check and then fails inside tf.transpose; here it
    raises ValueError when the layer is built."""

    def __init__(self, k=1, axis=-1, **kwargs):
        self.k = k
        self.axis = axis
        Layer.__init__(self, **kwargs)

    def build(self, input_shape):
        if self.axis < 1 or self.axis > len(input_shape):
            raise ValueError("axis must be 1~%d,now is %d" % (len(input_shape), self.axis))
        if self.axis == len(input_shape):
            raise ValueError("axis must be 1~%d,now is %d: axis %d is past the last axis of a %d-D input"
                             % (len(input_shape) - 1, self.axis, self.axis, len(input_shape)))
        if self.k < 1 or self.k > input_shape[self.axis]:
            raise ValueError("k must be in 1 ~ %d,now k is %d" % (input_shape[self.axis], self.k))
        self.dims = len(input_shape)
        K.conv_stack_check(int(input_shape[self.axis]), 1, [("kmax", self.k)])
        self.built = True

    def stage(self):
        return ("kmax", self.k)

    def call(self, inputs, **kwargs):
        shape = tuple(inputs.data.shape)
        n = shape[self.axis]
        inner = int(np.prod(shape[self.axis + 1:])) if self.axis + 1 < len(shape) else 1
        out_shape = shape[:self.axis] + (self.k,) + shape[self.axis + 1:]
        return ops.conv_stack(inputs, [self.stage()], n, inner, 1, out_shape)

    def compute_output_shape(self, input_shape):
        output_shape = list(input_shape)
        output_shape[self.axis] = self.k
        return tuple(output_shape)

    def get_config(self):
        config = {'k': self.k, 'axis': self.axis}
        base = Layer.get_config(self)
        base.update(config)
        return base
