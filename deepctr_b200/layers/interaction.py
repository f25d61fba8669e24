"""Host mirror of deepctr/layers/interaction.py for the operators on the hot path:
AFMLayer (:39-160), BiInteractionPooling (:163-206), FM (:563-607), CrossNet (:344-435), CIN (:209-341),
InteractingLayer (:697-790), SENETLayer (:1067-1139), BilinearInteraction (:1142-1221), FwFMLayer (:1350-1425),
FEFMLayer (:1428-1499), InnerProductLayer (:610-695), OutterProductLayer (:793-931), BridgeModule (:1502-1570),
FieldWiseBiInteraction (:1224-1348).
Same constructor arguments, weight names, shape checks and error messages as the reference."""
import itertools

import torch

from .. import engine as E
from .. import kernels as K
from .. import ops
from ..engine import Layer, Lambda, Zeros, Ones, Constant, glorot_normal, glorot_uniform, TruncatedNormal, l2
from .normalization import Dropout

# shapes the fused AFM kernels serve (include/b2ctr.h, b2ctr_afm_fwd)
AFM_MAX_FIELDS, AFM_MAX_EMBEDDING, AFM_MAX_FACTOR = 64, 32, 16
# shapes the SENET / bilinear kernels serve (include/b2ctr.h, b2ctr_senet_fwd, b2ctr_bilinear_fwd)
SENET_MAX_FIELDS, BILINEAR_MAX_FIELDS, BILINEAR_MAX_EMBEDDING = 64, 64, 64
# shapes the FwFM / FEFM kernels serve (include/b2ctr.h, b2ctr_fwfm_fwd, b2ctr_fefm_fwd)
FWFM_MAX_FIELDS, FWFM_MAX_EMBEDDING = 64, 64
FEFM_MAX_FIELDS, FEFM_MAX_EMBEDDING = 64, 64
# shapes the PNN product kernels serve (include/b2ctr.h, b2ctr_pnn_inner_fwd, b2ctr_pnn_outer_fwd)
PNN_MAX_FIELDS, PNN_MAX_EMBEDDING = 64, 64
# shapes the InteractingLayer attention kernels serve (include/b2ctr.h, b2ctr_interacting_fwd / _bwd)
INTERACTING_MAX_FIELDS, INTERACTING_MAX_ATT_EMBEDDING, INTERACTING_MAX_FHD = 64, 32, 3072


def _weights_stacked(layer, ws):
    """(ws, stack): the weights' device data as views of one [n, E, E] buffer ``layer._stack``, rebuilt when a
    weight's data is no longer its view (first call, set_value, loading).  The weights stay separate weights for
    set_value, loading by name and the optimizers; the kernels take the stack."""
    st = layer._stack
    if st is None or ws[0].data is None or ws[0].data.data_ptr() != st.data_ptr() or ws[-1].data is None \
            or ws[-1].data.data_ptr() != st[-1].data_ptr():
        st = torch.stack([w.materialize() for w in ws])
        for k, w in enumerate(ws):
            w.data = st[k]
        layer._stack = st
    return ws, st


class AFMLayer(Layer):
    """Attentional FM pooling, deepctr/layers/interaction.py:39-160.  Called on a list of F [B,1,E] tensors;
    att = sum_p softmax_p(h . relu(W^T (v_i * v_j) + b)) (v_i * v_j) over the pairs i < j, then
    out = Dropout(att) . projection_p  [B,1].  The pairwise products are generated inside the kernel
    (b2ctr_afm_fwd / _bwd): nothing of size [B, F(F-1)/2, .] is stored."""

    def __init__(self, attention_factor=4, l2_reg_w=0, dropout_rate=0, seed=1024, **kwargs):
        self.attention_factor = attention_factor
        self.l2_reg_w = l2_reg_w
        self.dropout_rate = dropout_rate
        self.seed = seed
        Layer.__init__(self, **kwargs)

    def build(self, input_shape):
        if not isinstance(input_shape, list) or len(input_shape) < 2:
            raise ValueError('A `AttentionalFM` layer should be called '
                             'on a list of at least 2 inputs')
        shape_set = set(tuple(s) for s in input_shape)
        if len(shape_set) > 1:
            raise ValueError('A `AttentionalFM` layer requires '
                             'inputs with same shapes '
                             'Got different shapes: %s' % (shape_set))
        if len(input_shape[0]) != 3 or input_shape[0][1] != 1:
            raise ValueError('A `AttentionalFM` layer requires '
                             'inputs of a list with same shape tensor like\
                             (None, 1, embedding_size)'
                             'Got different shapes: %s' % (input_shape[0],))
        embedding_size = int(input_shape[0][-1])
        if (len(input_shape) > AFM_MAX_FIELDS or embedding_size > AFM_MAX_EMBEDDING
                or not 1 <= int(self.attention_factor) <= AFM_MAX_FACTOR):
            raise ValueError("AFMLayer supports up to %d inputs, embedding_size <= %d and 1 <= attention_factor <= %d "
                             "(got %d inputs, embedding_size %d, attention_factor %r)"
                             % (AFM_MAX_FIELDS, AFM_MAX_EMBEDDING, AFM_MAX_FACTOR, len(input_shape),
                                embedding_size, self.attention_factor))
        self.attention_W = self.add_weight(shape=(embedding_size, self.attention_factor),
                                           initializer=glorot_normal(seed=self.seed),
                                           regularizer=l2(self.l2_reg_w), name="attention_W")
        self.attention_b = self.add_weight(shape=(self.attention_factor,), initializer=Zeros(), name="attention_b")
        self.projection_h = self.add_weight(shape=(self.attention_factor, 1),
                                            initializer=glorot_normal(seed=self.seed), name="projection_h")
        self.projection_p = self.add_weight(shape=(embedding_size, 1), initializer=glorot_normal(seed=self.seed),
                                            name="projection_p")
        # the reference creates these two layers here: they take the next `dropout` / `lambda` names
        self.dropout = self._track(Dropout(self.dropout_rate, seed=self.seed, name=self.name + "/dropout"))
        self.tensordot = self._track(Lambda(lambda x: ops.dense(x[0], x[1]), name=self.name + "/tensordot"))
        self.built = True

    def call(self, inputs, training=None, **kwargs):
        if inputs[0].data.dim() != 3:
            raise ValueError("Unexpected inputs dimensions %d, expect to be 3 dimensions" % (inputs[0].data.dim()))
        fields = ops.concat(inputs, axis=1)             # a zero-copy window of the fused gather's buffer
        att = ops.afm(fields, self.attention_W, self.attention_b, self.projection_h)
        att = self.dropout.call(att, training=training)
        return self.tensordot.call([att, self.projection_p])

    def compute_output_shape(self, input_shape):
        if not isinstance(input_shape, list):
            raise ValueError('A `AFMLayer` layer should be called '
                             'on a list of inputs.')
        return (None, 1)

    def get_config(self):
        config = {'attention_factor': self.attention_factor,
                  'l2_reg_w': self.l2_reg_w, 'dropout_rate': self.dropout_rate, 'seed': self.seed}
        base = Layer.get_config(self)
        base.update(config)
        return base


class BiInteractionPooling(Layer):
    """Bi-Interaction pooling of NFM, deepctr/layers/interaction.py:163-206.
    [B,F,E] -> [B,1,E]:  0.5 * ((sum_f x)^2 - sum_f x^2)  (FM without the final sum over E)."""

    def build(self, input_shape):
        if len(input_shape) != 3:
            raise ValueError("Unexpected inputs dimensions %d, expect to be 3 dimensions" % (len(input_shape)))
        self.built = True

    def call(self, inputs, **kwargs):
        if inputs.data.dim() != 3:
            raise ValueError("Unexpected inputs dimensions %d, expect to be 3 dimensions" % (inputs.data.dim()))
        return ops.bi_interaction(inputs)

    def compute_output_shape(self, input_shape):
        return (None, 1, input_shape[-1])


class FM(Layer):
    """Factorization Machine second-order term, deepctr/layers/interaction.py:563-607.
    [B,F,E] -> [B,1].  When the input is the fused gather's buffer the value comes out of the gather
    kernel's epilogue (no extra pass over [B,F,E]).  IFM / DIFM's refined input x * m reaches it as its two factors
    (ops.ScaledFields) and runs the field-weighted FM: the product is never written."""
    takes_scaled_fields = True

    def build(self, input_shape):
        if len(input_shape) != 3:
            raise ValueError("Unexpected inputs dimensions % d,\
                             expect to be 3 dimensions" % (len(input_shape)))
        self.built = True

    def call(self, inputs, **kwargs):
        if len(inputs.shape) != 3:
            raise ValueError("Unexpected inputs dimensions %d, expect to be 3 dimensions" % (len(inputs.shape)))
        planner = getattr(self, "_planner", None)
        if planner is not None and not isinstance(inputs, ops.ScaledFields):
            fused = planner.lookup_fm(inputs)
            if fused is not None:
                return fused
        return ops.fm(inputs)

    def compute_output_shape(self, input_shape):
        return (None, 1)


class CrossNet(Layer):
    """deepctr/layers/interaction.py:344-435.  vector: x_{l+1} = x_0 (x_l . w_l) + b_l + x_l;
    matrix: x_{l+1} = x_0 * (W_l x_l + b_l) + x_l."""

    def __init__(self, layer_num=2, parameterization='vector', l2_reg=0, seed=1024, **kwargs):
        self.layer_num = layer_num
        self.parameterization = parameterization
        self.l2_reg = l2_reg
        self.seed = seed
        print('CrossNet parameterization:', self.parameterization)
        Layer.__init__(self, **kwargs)

    def build(self, input_shape):
        if len(input_shape) != 2:
            raise ValueError("Unexpected inputs dimensions %d, expect to be 2 dimensions" % (len(input_shape),))
        dim = int(input_shape[-1])
        if self.parameterization == 'vector':
            shape = (dim, 1)
        elif self.parameterization == 'matrix':
            shape = (dim, dim)
        else:
            raise ValueError("parameterization should be 'vector' or 'matrix'")
        self.kernels = [self.add_weight(name='kernel' + str(i), shape=shape,
                                        initializer=glorot_normal(seed=self.seed),
                                        regularizer=l2(self.l2_reg), trainable=True)
                        for i in range(self.layer_num)]
        self.bias = [self.add_weight(name='bias' + str(i), shape=(dim, 1), initializer=Zeros(), trainable=True)
                     for i in range(self.layer_num)]
        self.built = True

    def call(self, inputs, **kwargs):
        if inputs.data.dim() != 2:
            raise ValueError("Unexpected inputs dimensions %d, expect to be 2 dimensions" % (inputs.data.dim()))
        x_0 = inputs
        x_l = x_0
        for i in range(self.layer_num):
            if self.parameterization == 'vector':
                x_l = ops.cross_vector(x_0, x_l, self.kernels[i], self.bias[i])
            else:
                x_l = ops.cross_matrix(x_0, x_l, self.kernels[i], self.bias[i])
        return x_l

    def get_config(self):
        config = {'layer_num': self.layer_num, 'parameterization': self.parameterization,
                  'l2_reg': self.l2_reg, 'seed': self.seed}
        base = Layer.get_config(self)
        base.update(config)
        return base

    def compute_output_shape(self, input_shape):
        return input_shape


class CIN(Layer):
    """Compressed Interaction Network, deepctr/layers/interaction.py:209-341.
    out[b,d,n] = act(sum_{i,j} X0[b,i,d] * Xk[b,j,d] * W_k[i*H_k + j, n] + bias_k[n]); the
    [B, D, m*H_k] outer product of the reference (:291-297) is never materialised."""

    def __init__(self, layer_size=(128, 128), activation='relu', split_half=True, l2_reg=1e-5, seed=1024,
                 **kwargs):
        if len(layer_size) == 0:
            raise ValueError("layer_size must be a list(tuple) of length greater than 1")
        self.layer_size = layer_size
        self.split_half = split_half
        self.activation = activation
        self.l2_reg = l2_reg
        self.seed = seed
        Layer.__init__(self, **kwargs)

    def build(self, input_shape):
        if len(input_shape) != 3:
            raise ValueError("Unexpected inputs dimensions %d, expect to be 3 dimensions" % (len(input_shape)))
        self.field_nums = [int(input_shape[1])]
        self.filters = []
        self.bias = []
        for i, size in enumerate(self.layer_size):
            self.filters.append(self.add_weight(name='filter' + str(i),
                                                shape=[1, self.field_nums[-1] * self.field_nums[0], size],
                                                initializer=glorot_uniform(seed=self.seed + i),
                                                regularizer=l2(self.l2_reg)))
            self.bias.append(self.add_weight(name='bias' + str(i), shape=[size], initializer=Zeros()))
            if self.split_half:
                if i != len(self.layer_size) - 1 and size % 2 > 0:
                    raise ValueError(
                        "layer_size must be even number except for the last layer when split_half=True")
                self.field_nums.append(size // 2)
            else:
                self.field_nums.append(size)
        from .activation import fusable_activation
        if not fusable_activation(self.activation):
            raise ValueError("CIN activation %r is not supported" % (self.activation,))
        self.built = True

    def call(self, inputs, **kwargs):
        if inputs.data.dim() != 3:
            raise ValueError("Unexpected inputs dimensions %d, expect to be 3 dimensions" % (inputs.data.dim()))
        return ops.cin(inputs, self.filters, self.bias, self.layer_size, self.activation, self.split_half)

    def compute_output_shape(self, input_shape):
        if self.split_half:
            featuremap_num = sum(self.layer_size[:-1]) // 2 + self.layer_size[-1]
        else:
            featuremap_num = sum(self.layer_size)
        return (None, featuremap_num)

    def get_config(self):
        config = {'layer_size': self.layer_size, 'split_half': self.split_half, 'activation': self.activation,
                  'seed': self.seed}
        base = Layer.get_config(self)
        base.update(config)
        return base


class InteractingLayer(Layer):
    """AutoInt multi-head self-attention over fields, deepctr/layers/interaction.py:697-790."""

    def __init__(self, att_embedding_size=8, head_num=2, use_res=True, scaling=False, seed=1024, **kwargs):
        if head_num <= 0:
            raise ValueError('head_num must be a int > 0')
        self.att_embedding_size = att_embedding_size
        self.head_num = head_num
        self.use_res = use_res
        self.seed = seed
        self.scaling = scaling
        Layer.__init__(self, **kwargs)

    def build(self, input_shape):
        if len(input_shape) != 3:
            raise ValueError("Unexpected inputs dimensions %d, expect to be 3 dimensions" % (len(input_shape)))
        embedding_size = int(input_shape[-1])
        n = self.att_embedding_size * self.head_num
        fields = input_shape[1]
        if (fields is not None and int(fields) > INTERACTING_MAX_FIELDS
                or self.att_embedding_size > INTERACTING_MAX_ATT_EMBEDDING
                or fields is not None and int(fields) * n > INTERACTING_MAX_FHD):
            raise ValueError("InteractingLayer supports up to %d fields, att_embedding_size <= %d and "
                             "fields * head_num * att_embedding_size <= %d (got %s fields, head_num %d, "
                             "att_embedding_size %d)" % (INTERACTING_MAX_FIELDS, INTERACTING_MAX_ATT_EMBEDDING,
                                                         INTERACTING_MAX_FHD, fields, self.head_num,
                                                         self.att_embedding_size))
        self.W_Query = self.add_weight(name='query', shape=[embedding_size, n],
                                       initializer=TruncatedNormal(seed=self.seed))
        self.W_key = self.add_weight(name='key', shape=[embedding_size, n],
                                     initializer=TruncatedNormal(seed=self.seed + 1))
        self.W_Value = self.add_weight(name='value', shape=[embedding_size, n],
                                       initializer=TruncatedNormal(seed=self.seed + 2))
        if self.use_res:
            self.W_Res = self.add_weight(name='res', shape=[embedding_size, n],
                                         initializer=TruncatedNormal(seed=self.seed))
        self.built = True

    def call(self, inputs, **kwargs):
        if inputs.data.dim() != 3:
            raise ValueError("Unexpected inputs dimensions %d, expect to be 3 dimensions" % (inputs.data.dim()))
        querys = ops.dense(inputs, self.W_Query)
        keys = ops.dense(inputs, self.W_key)
        values = ops.dense(inputs, self.W_Value)
        res = ops.dense(inputs, self.W_Res) if self.use_res else None
        return ops.interacting_attention(querys, keys, values, res, self.head_num, self.att_embedding_size,
                                         self.scaling)

    def compute_output_shape(self, input_shape):
        return (None, input_shape[1], self.att_embedding_size * self.head_num)

    def get_config(self):
        config = {'att_embedding_size': self.att_embedding_size, 'head_num': self.head_num,
                  'use_res': self.use_res, 'seed': self.seed}
        base = Layer.get_config(self)
        base.update(config)
        return base


class SENETLayer(Layer):
    """SENET of FiBiNET, deepctr/layers/interaction.py:1067-1139.  Called on a list of F [B,1,E] tensors; returns F
    [B,1,E] windows of V = x * relu(relu(mean_e(x) W_1) W_2)[:, :, None] (b2ctr_senet_fwd / _bwd: the input is read
    in place, only V and the [B, R + F] excitation are written)."""

    def __init__(self, reduction_ratio=3, seed=1024, **kwargs):
        self.reduction_ratio = reduction_ratio
        self.seed = seed
        Layer.__init__(self, **kwargs)

    def build(self, input_shape):
        if not isinstance(input_shape, list) or len(input_shape) < 2:
            raise ValueError('A `AttentionalFM` layer should be called '
                             'on a list of at least 2 inputs')
        self.filed_size = len(input_shape)
        self.embedding_size = input_shape[0][-1]
        reduction_size = max(1, self.filed_size // self.reduction_ratio)
        if self.filed_size > SENET_MAX_FIELDS or not 1 <= reduction_size <= SENET_MAX_FIELDS:
            raise ValueError("SENETLayer supports up to %d inputs and a reduction size of 1 to %d "
                             "(got %d inputs, reduction size %r)"
                             % (SENET_MAX_FIELDS, SENET_MAX_FIELDS, self.filed_size, reduction_size))
        self.W_1 = self.add_weight(shape=(self.filed_size, reduction_size), initializer=glorot_normal(seed=self.seed),
                                   name="W_1")
        self.W_2 = self.add_weight(shape=(reduction_size, self.filed_size), initializer=glorot_normal(seed=self.seed),
                                   name="W_2")
        # the reference creates this layer here: it takes the next `lambda` name
        self.tensordot = self._track(Lambda(lambda x: ops.dense(x[0], x[1]), name=self.name + "/tensordot"))
        self.built = True

    def call(self, inputs, training=None, **kwargs):
        if inputs[0].data.dim() != 3:
            raise ValueError("Unexpected inputs dimensions %d, expect to be 3 dimensions" % (inputs[0].data.dim()))
        x = ops.concat(inputs, axis=1)           # a zero-copy window of the fused gather's buffer
        b, f, e = x.data.shape
        v = ops.senet(x, self.W_1, self.W_2)
        return [ops._window(v, i * e, e, (b, 1, e)) for i in range(f)]

    def compute_output_shape(self, input_shape):
        return input_shape

    def compute_mask(self, inputs, mask=None):
        return [None] * self.filed_size

    def get_config(self):
        config = {'reduction_ratio': self.reduction_ratio, 'seed': self.seed}
        base = Layer.get_config(self)
        base.update(config)
        return base


class BilinearInteraction(Layer):
    """Bilinear interaction of FiBiNET, deepctr/layers/interaction.py:1142-1221.  Called on a list of F [B,1,E]
    tensors; output [B, P, E] with row p = (i < j) equal to (v_i W) * v_j, W one weight ('all'), one per first field
    ('each') or one per pair ('interaction').  The weights keep the reference's names and order but their data are
    views of one stacked [nW, E, E] buffer, which is what b2ctr_bilinear_fwd / _bwd take.  When the model's graph
    lets it (inputs.DnnInputPlacement), the pairs are written straight into the first DNN layer's input."""

    def __init__(self, bilinear_type="interaction", seed=1024, **kwargs):
        self.bilinear_type = bilinear_type
        self.seed = seed
        self._stack = None
        Layer.__init__(self, **kwargs)

    def build(self, input_shape):
        if not isinstance(input_shape, list) or len(input_shape) < 2:
            raise ValueError('A `AttentionalFM` layer should be called '
                             'on a list of at least 2 inputs')
        embedding_size = int(input_shape[0][-1])
        if len(input_shape) > BILINEAR_MAX_FIELDS or embedding_size > BILINEAR_MAX_EMBEDDING:
            raise ValueError("BilinearInteraction supports up to %d inputs and embedding_size <= %d "
                             "(got %d inputs, embedding_size %d)"
                             % (BILINEAR_MAX_FIELDS, BILINEAR_MAX_EMBEDDING, len(input_shape), embedding_size))
        shape = (embedding_size, embedding_size)
        if self.bilinear_type == "all":
            self.W = self.add_weight(shape=shape, initializer=glorot_normal(seed=self.seed), name="bilinear_weight")
        elif self.bilinear_type == "each":
            self.W_list = [self.add_weight(shape=shape, initializer=glorot_normal(seed=self.seed),
                                           name="bilinear_weight" + str(i)) for i in range(len(input_shape) - 1)]
        elif self.bilinear_type == "interaction":
            self.W_list = [self.add_weight(shape=shape, initializer=glorot_normal(seed=self.seed),
                                           name="bilinear_weight" + str(i) + '_' + str(j))
                           for i, j in itertools.combinations(range(len(input_shape)), 2)]
        else:
            raise NotImplementedError
        self.built = True

    def call(self, inputs, **kwargs):
        if inputs[0].data.dim() != 3:
            raise ValueError("Unexpected inputs dimensions %d, expect to be 3 dimensions" % (inputs[0].data.dim()))
        if self.bilinear_type not in ("all", "each", "interaction"):
            raise NotImplementedError
        x = ops.concat(inputs, axis=1)
        ws, st = _weights_stacked(self, [self.W] if self.bilinear_type == "all" else self.W_list)
        planner = getattr(self, "_planner", None)
        place = planner.dnn_input_place(self) if planner is not None else None
        if place is None:
            return ops.bilinear_interaction(x, ws, st, self.bilinear_type)
        pl, k = place
        b, f, e = x.data.shape
        out = ops.bilinear_interaction(x, ws, st, self.bilinear_type, out=pl.out_view(k, b, x.data.device))
        pl.placed(k, out)
        return out

    def compute_output_shape(self, input_shape):
        filed_size = len(input_shape)
        embedding_size = input_shape[0][-1]
        return (None, filed_size * (filed_size - 1) // 2, embedding_size)

    def get_config(self):
        config = {'bilinear_type': self.bilinear_type, 'seed': self.seed}
        base = Layer.get_config(self)
        base.update(config)
        return base


class FwFMLayer(Layer):
    """Field-weighted FM, deepctr/layers/interaction.py:1350-1425.  Called on a [B, F, E] tensor; output [B, 1] =
    sum_{i<j} r[i, j] <x_i, x_j> with the [F, F] field_pair_strengths r, of which only the upper triangle is read
    (b2ctr_fwfm_fwd / _bwd: the input is read in place; the gradient of r is 0 on and below the diagonal)."""

    def __init__(self, num_fields=4, regularizer=0.000001, **kwargs):
        self.num_fields = num_fields
        self.regularizer = regularizer
        Layer.__init__(self, **kwargs)

    def build(self, input_shape):
        if len(input_shape) != 3:
            raise ValueError("Unexpected inputs dimensions % d,                             expect to be 3 dimensions"
                             % (len(input_shape)))
        if input_shape[1] != self.num_fields:
            raise ValueError("Mismatch in number of fields {} and                  concatenated embeddings dims {}"
                             .format(self.num_fields, input_shape[1]))
        embedding_size = int(input_shape[2])
        if not 2 <= self.num_fields <= FWFM_MAX_FIELDS or not 1 <= embedding_size <= FWFM_MAX_EMBEDDING:
            raise ValueError("FwFMLayer supports 2 to %d fields and embedding_size 1 to %d "
                             "(got %d fields, embedding_size %d)"
                             % (FWFM_MAX_FIELDS, FWFM_MAX_EMBEDDING, self.num_fields, embedding_size))
        self.field_strengths = self.add_weight(name='field_pair_strengths', shape=(self.num_fields, self.num_fields),
                                               initializer=TruncatedNormal(), regularizer=l2(self.regularizer),
                                               trainable=True)
        self.built = True

    def call(self, inputs, **kwargs):
        if inputs.data.dim() != 3:
            raise ValueError("Unexpected inputs dimensions %d, expect to be 3 dimensions" % (inputs.data.dim()))
        if inputs.data.shape[1] != self.num_fields:
            raise ValueError("Mismatch in number of fields {} and                  concatenated embeddings dims {}"
                             .format(self.num_fields, inputs.data.shape[1]))
        return ops.fwfm(inputs, self.field_strengths)

    def compute_output_shape(self, input_shape):
        return (None, 1)

    def get_config(self):
        config = Layer.get_config(self).copy()
        config.update({'num_fields': self.num_fields, 'regularizer': self.regularizer})
        return config


class FEFMLayer(Layer):
    """Field-embedded FM, deepctr/layers/interaction.py:1428-1499.  Called on a [B, F, E] tensor; output [B, P] with
    column p = (i < j) equal to x_i (W_p + W_p^T) x_j^T.  The P weights field_embeddings{i}-{j} keep the reference's
    names and order but their data are views of one stacked [P, E, E] buffer, which is what b2ctr_fefm_sym / _fwd /
    _bwd take.  In DeepFEFM the scores are written straight into the first DNN layer's input
    (inputs.EmbeddingPlanner.fefm_place)."""

    def __init__(self, regularizer, **kwargs):
        self.regularizer = regularizer
        self._stack = None
        Layer.__init__(self, **kwargs)

    def build(self, input_shape):
        if len(input_shape) != 3:
            raise ValueError("Unexpected inputs dimensions % d,                                expect to be 3 "
                             "dimensions" % (len(input_shape)))
        self.num_fields = int(input_shape[1])
        embedding_size = int(input_shape[2])
        if not 2 <= self.num_fields <= FEFM_MAX_FIELDS or not 1 <= embedding_size <= FEFM_MAX_EMBEDDING:
            raise ValueError("FEFMLayer supports 2 to %d fields and embedding_size 1 to %d "
                             "(got %d fields, embedding_size %d)"
                             % (FEFM_MAX_FIELDS, FEFM_MAX_EMBEDDING, self.num_fields, embedding_size))
        self.field_embeddings = {}
        for fi, fj in itertools.combinations(range(self.num_fields), 2):
            field_pair_id = str(fi) + "-" + str(fj)
            self.field_embeddings[field_pair_id] = self.add_weight(name='field_embeddings' + field_pair_id,
                                                                   shape=(embedding_size, embedding_size),
                                                                   initializer=TruncatedNormal(),
                                                                   regularizer=l2(self.regularizer),
                                                                   trainable=True)
        self.built = True

    def call(self, inputs, **kwargs):
        if inputs.data.dim() != 3:
            raise ValueError("Unexpected inputs dimensions %d, expect to be 3 dimensions" % (inputs.data.dim()))
        ws, st = _weights_stacked(self, list(self.field_embeddings.values()))
        planner = getattr(self, "_planner", None)
        out = planner.fefm_place(self, inputs) if planner is not None else None
        return ops.fefm(inputs, ws, st, out=out)

    def compute_output_shape(self, input_shape):
        # the reference divides with `/` (a float); the graph here needs the integer column count
        num_fields = int(input_shape[1])
        return (None, (num_fields * (num_fields - 1)) // 2)

    def get_config(self):
        config = Layer.get_config(self).copy()
        config.update({'regularizer': self.regularizer})
        return config


def _check_product_inputs(name, input_shape):
    """The reference's list-of-[B,1,E] checks and messages (InnerProductLayer / OutterProductLayer.build), then the
    kernels' limits."""
    if not isinstance(input_shape, list) or len(input_shape) < 2:
        raise ValueError('A `%s` layer should be called '
                         'on a list of at least 2 inputs' % name)
    shape_set = set(tuple(s) for s in input_shape)
    if len(shape_set) > 1:
        raise ValueError('A `%s` layer requires '
                         'inputs with same shapes '
                         'Got different shapes: %s' % (name, shape_set))
    if len(input_shape[0]) != 3 or input_shape[0][1] != 1:
        raise ValueError('A `%s` layer requires '
                         'inputs of a list with same shape tensor like (None,1,embedding_size)'
                         'Got different shapes: %s' % (name, input_shape[0]))
    num_inputs, embed_size = len(input_shape), int(input_shape[0][-1])
    if num_inputs > PNN_MAX_FIELDS or not 1 <= embed_size <= PNN_MAX_EMBEDDING:
        raise ValueError("%s supports 2 to %d inputs and embedding_size 1 to %d (got %d inputs, embedding_size %d)"
                         % (name, PNN_MAX_FIELDS, PNN_MAX_EMBEDDING, num_inputs, embed_size))
    return num_inputs, embed_size


def _product_place(layer, x):
    planner = getattr(layer, "_planner", None)
    return planner.pnn_place(layer, x) if planner is not None else None


def _product_operand(inputs):
    if inputs[0].data.dim() != 3:
        raise ValueError("Unexpected inputs dimensions %d, expect to be 3 dimensions" % (inputs[0].data.dim()))
    # consecutive windows of the gather buffer concatenate to a zero-copy [B, F, E] window; anything else is one copy
    return ops.concat(inputs, axis=1)


class InnerProductLayer(Layer):
    """PNN's inner products, deepctr/layers/interaction.py:610-695.  Called on a list of F [B,1,E] tensors; output
    [B, P, 1] with row p = (i < j) equal to <v_i, v_j> (reduce_sum=True), or [B, P, E] with v_i * v_j
    (b2ctr_pnn_inner_fwd: the gather buffer is read in place and no per-pair [B, E] product is written for the
    inner products).  In PNN the products are written straight into the first DNN layer's input
    (inputs.EmbeddingPlanner.pnn_place)."""

    def __init__(self, reduce_sum=True, **kwargs):
        self.reduce_sum = reduce_sum
        Layer.__init__(self, **kwargs)

    def build(self, input_shape):
        _check_product_inputs("InnerProductLayer", input_shape)
        self.built = True

    def call(self, inputs, **kwargs):
        x = _product_operand(inputs)
        if not self.reduce_sum:
            return ops.pnn_inner(x, "elementwise")
        return ops.pnn_inner(x, "inner", out=_product_place(self, x))

    def compute_output_shape(self, input_shape):
        num_inputs = len(input_shape)
        num_pairs = num_inputs * (num_inputs - 1) // 2
        input_shape = input_shape[0]
        return (input_shape[0], num_pairs, 1 if self.reduce_sum else input_shape[-1])

    def get_config(self):
        config = {'reduce_sum': self.reduce_sum}
        base_config = Layer.get_config(self)
        base_config.update(config)
        return base_config


class OutterProductLayer(Layer):
    """PNN's outer products, deepctr/layers/interaction.py:793-931.  Called on a list of F [B,1,E] tensors; output
    [B, P] with, for the pair p = (i < j), sum_{k,l} v_j[k] K[k,p,l] v_i[l] (kernel_type 'mat', K [E,P,E], on the
    FEFM tiles: b2ctr_pnn_outer_fwd), sum_e v_i[e] v_j[e] K[p,e] ('vec', K [P,E]) or K[p] <v_i, v_j> ('num', K [P,1])
    (b2ctr_pnn_inner_fwd).  The weight keeps the reference's name, shape and glorot_uniform(seed) initialiser."""

    def __init__(self, kernel_type='mat', seed=1024, **kwargs):
        if kernel_type not in ['mat', 'vec', 'num']:
            raise ValueError("kernel_type must be mat,vec or num")
        self.kernel_type = kernel_type
        self.seed = seed
        Layer.__init__(self, **kwargs)

    def build(self, input_shape):
        num_inputs, embed_size = _check_product_inputs("OutterProductLayer", input_shape)
        num_pairs = num_inputs * (num_inputs - 1) // 2
        if self.kernel_type == 'mat':
            self.kernel = self.add_weight(shape=(embed_size, num_pairs, embed_size),
                                          initializer=glorot_uniform(seed=self.seed), name='kernel')
        elif self.kernel_type == 'vec':
            self.kernel = self.add_weight(shape=(num_pairs, embed_size,), initializer=glorot_uniform(self.seed),
                                          name='kernel')
        elif self.kernel_type == 'num':
            self.kernel = self.add_weight(shape=(num_pairs, 1), initializer=glorot_uniform(self.seed), name='kernel')
        self.built = True

    def call(self, inputs, **kwargs):
        x = _product_operand(inputs)
        out = _product_place(self, x)
        if self.kernel_type == 'mat':
            return ops.pnn_outer(x, self.kernel, out=out)
        return ops.pnn_inner(x, self.kernel_type, self.kernel, out=out)

    def compute_output_shape(self, input_shape):
        num_inputs = len(input_shape)
        return (None, num_inputs * (num_inputs - 1) // 2)

    def get_config(self):
        config = {'kernel_type': self.kernel_type, 'seed': self.seed}
        base_config = Layer.get_config(self)
        base_config.update(config)
        return base_config


BRIDGE_TYPES = ("pointwise_addition", "hadamard_product", "concatenation", "attention_pooling")
# b2ctr_regulate mode of each bridge type it serves; 'concatenation' is Concatenate + Dense on the GEMM
_BRIDGE_MODES = {"pointwise_addition": "add", "hadamard_product": "hadamard", "attention_pooling": "attention"}


class BridgeModule(Layer):
    """EDCN's bridge between the cross and deep stacks, deepctr/layers/interaction.py:1502-1570.  Called on
    [x, h], two [B, d] tensors: x + h ('pointwise_addition'), x * h ('hadamard_product'), Dense(d, activation)
    of concat([x, h]) ('concatenation') or a_x * x + a_h * h with a_x = DNN([d, d], activation,
    output_activation='softmax')(x) and a_h likewise of h ('attention_pooling').  The nested Dense / DNNs are created
    in build() and take Keras' automatic names.  Except for 'concatenation' the bridge is one b2ctr_regulate launch;
    when its output only feeds two RegulationModules through a Reshape, the planner (inputs.RegulatePlan) makes that
    launch write the two gated outputs instead, and the bridge output itself is never written.

    Deviation: an unknown ``bridge_type`` raises ValueError here; the reference's call returns None and fails later
    inside TensorFlow."""

    def __init__(self, bridge_type='hadamard_product', activation='relu', **kwargs):
        if bridge_type not in BRIDGE_TYPES:
            raise ValueError("BridgeModule bridge_type %r is not one of %s" % (bridge_type, ", ".join(BRIDGE_TYPES)))
        self.bridge_type = bridge_type
        self.activation = activation
        Layer.__init__(self, **kwargs)

    def build(self, input_shape):
        if not isinstance(input_shape, list) or len(input_shape) < 2:
            raise ValueError('A `BridgeModule` layer should be called '
                             'on a list of 2 inputs')
        self.dnn_dim = int(input_shape[0][-1])
        from .core import DNN
        if self.bridge_type == "concatenation":
            self.dense = self._track(E.Dense(self.dnn_dim, self.activation, name=self.name + "/dense"))
            self.dense._maybe_build((None, 2 * self.dnn_dim))
        elif self.bridge_type == "attention_pooling":
            self.dense_x = self._track(DNN([self.dnn_dim, self.dnn_dim], self.activation, output_activation='softmax',
                                           name=self.name + "/dense_x"))
            self.dense_h = self._track(DNN([self.dnn_dim, self.dnn_dim], self.activation, output_activation='softmax',
                                           name=self.name + "/dense_h"))
            self.dense_x._maybe_build(tuple(input_shape[0]))
            self.dense_h._maybe_build(tuple(input_shape[1]))
        self.built = True

    def call(self, inputs, training=None, **kwargs):
        x, h = inputs
        if self.bridge_type == "concatenation":
            return self.dense.call(ops.concat([x, h], axis=-1))
        ax = ah = None
        if self.bridge_type == "attention_pooling":
            ax = self.dense_x.call(x, training=training)
            ah = self.dense_h.call(h, training=training)
        mode = _BRIDGE_MODES[self.bridge_type]
        planner = getattr(self, "_planner", None)
        served = planner.bridged(self, mode, (x, h, ax, ah)) if planner is not None else None
        if served is not None:
            return served
        u, _ = ops.regulate(mode, x, h, ax, ah)
        return u

    def compute_output_shape(self, input_shape):
        return (None, int(input_shape[0][-1]))

    def get_config(self):
        base = Layer.get_config(self).copy()
        config = {'bridge_type': self.bridge_type, 'activation': self.activation}
        config.update(base)
        return config


class FieldWiseBiInteraction(Layer):
    """FLEN's Field-Wise Bi-Interaction, deepctr/layers/interaction.py:1224-1348.  Called on a list of G >= 2
    [B, F_g, E] tensors (the field groups); output [B, E] =
      sum_{g<h} kernel_mf[p] * S_g * S_h + bias_mf + sum_g kernel_fm[g] * (S_g^2 - Q_g) + bias_fm
    with S_g / Q_g the sum / sum of squares of group g's fields.  One b2ctr_field_wise_bi launch: the groups are read
    wherever they are when they are windows of one buffer, else copied once into one [B, F, E] buffer.  In FLEN
    the planner (inputs.FieldWisePlan) hands it the group members, windows of the gather buffer, so the groups'
    concatenations are never written."""

    def __init__(self, use_bias=True, seed=1024, **kwargs):
        self.use_bias = use_bias
        self.seed = seed
        Layer.__init__(self, **kwargs)

    def build(self, input_shape):
        if not isinstance(input_shape, list) or len(input_shape) < 2:
            raise ValueError('A `Field-Wise Bi-Interaction` layer should be called '
                             'on a list of at least 2 inputs')
        self.num_fields = len(input_shape)
        embedding_size = int(input_shape[0][-1])
        nfield = sum(int(s[1]) for s in input_shape if len(s) == 3)
        K.field_wise_bi_check(nfield, self.num_fields, embedding_size)
        self.kernel_mf = self.add_weight(name='kernel_mf', shape=(int(self.num_fields * (self.num_fields - 1) / 2), 1),
                                         initializer=Ones(), regularizer=None, trainable=True)
        self.kernel_fm = self.add_weight(name='kernel_fm', shape=(self.num_fields, 1), initializer=Constant(value=0.5),
                                         regularizer=None, trainable=True)
        if self.use_bias:
            self.bias_mf = self.add_weight(name='bias_mf', shape=(embedding_size,), initializer=Zeros())
            self.bias_fm = self.add_weight(name='bias_fm', shape=(embedding_size,), initializer=Zeros())
        self.built = True

    def call(self, inputs, **kwargs):
        bias = (self.bias_mf, self.bias_fm) if self.use_bias else (None, None)
        planner = getattr(self, "_planner", None)
        groups = planner.field_wise_groups(self) if planner is not None else None
        if groups is None:
            if inputs[0].data.dim() != 3:
                raise ValueError("Unexpected inputs dimensions %d, expect to be 3 dimensions"
                                 % (inputs[0].data.dim()))
            groups = [[x] for x in inputs]
        return ops.field_wise_bi(groups, self.kernel_mf, self.kernel_fm, *bias)

    def compute_output_shape(self, input_shape):
        return (None, input_shape[0][-1])

    def get_config(self):
        config = {'use_bias': self.use_bias, 'seed': self.seed}
        base_config = Layer.get_config(self).copy()
        base_config.update(config)
        return base_config
