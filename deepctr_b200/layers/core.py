"""Host mirror of deepctr/layers/core.py: DNN (:123-223), PredictionLayer (:226-267),
LocalActivationUnit (:28-120), RegulationModule (:270-321)."""
from .. import _lib as L
from .. import engine as E
from .. import ops
from ..engine import Layer, Ones, Zeros, glorot_normal, l2
from .activation import activation_layer, fusable_activation


class DNN(Layer):
    """The Multi Layer Perceptron, deepctr/layers/core.py:123-223.

    Per layer: tensordot + bias -> [BatchNormalization] -> activation -> Dropout.  bias + activation
    are fused into the GEMM epilogue when the activation is relu / sigmoid / tanh / linear and no
    BatchNormalization sits in between."""

    def __init__(self, hidden_units, activation='relu', l2_reg=0, dropout_rate=0, use_bn=False,
                 output_activation=None, seed=1024, **kwargs):
        self.hidden_units = hidden_units
        self.activation = activation
        self.l2_reg = l2_reg
        self.dropout_rate = dropout_rate
        self.use_bn = use_bn
        self.output_activation = output_activation
        self.seed = seed
        Layer.__init__(self, **kwargs)

    def build(self, input_shape):
        input_size = input_shape[-1]
        hidden_units = [int(input_size)] + list(self.hidden_units)
        # same glorot_normal(seed) for every layer, as the reference (core.py:165-171)
        self.kernels = [self.add_weight(name='kernel' + str(i), shape=(hidden_units[i], hidden_units[i + 1]),
                                        initializer=glorot_normal(seed=self.seed),
                                        regularizer=l2(self.l2_reg), trainable=True)
                        for i in range(len(self.hidden_units))]
        self.bias = [self.add_weight(name='bias' + str(i), shape=(self.hidden_units[i],),
                                     initializer=Zeros(), trainable=True)
                     for i in range(len(self.hidden_units))]
        if self.use_bn:
            from .normalization import BatchNormalization
            self.bn_layers = [self._track(BatchNormalization(name=self.name + "/bn%d" % i))
                              for i in range(len(self.hidden_units))]
        from .normalization import Dropout
        self.dropout_layers = [Dropout(self.dropout_rate, seed=self.seed + i)
                               for i in range(len(self.hidden_units))]
        self.act_names = [self.output_activation if i == len(self.hidden_units) - 1 and self.output_activation
                          else self.activation for i in range(len(self.hidden_units))]
        self.activation_layers = [None if (fusable_activation(a) and not self.use_bn)
                                  else self._track(activation_layer(a, name=self.name + "/act%d" % i))
                                  for i, a in enumerate(self.act_names)]
        # build sub-layers now so that their weights exist (get_weights / set_weights) before the first call
        for i in range(len(self.hidden_units)):
            shape = tuple(input_shape[:-1]) + (int(self.hidden_units[i]),)
            if self.use_bn:
                self.bn_layers[i]._maybe_build(shape)
            if self.activation_layers[i] is not None:
                self.activation_layers[i]._maybe_build(shape)
        self.built = True

    def call(self, inputs, training=None, first=None, **kwargs):
        """``first(kernel, bias, activation)``: an alternative implementation of layer 0's  act(x W + b)  for a
        caller that never materialises x (the DIN attention unit generates it inside the GEMM)."""
        deep_input = inputs
        if (first is None and not self.use_bn and not (self.dropout_rate and training)
                and all(a == 'relu' for a in self.act_names)
                and ops.mlp_fusable(inputs, [int(u) for u in self.hidden_units])):
            # the whole relu tower as one tape node: layer 0's GEMM, then fused kernels for the layers after it
            return ops.mlp(inputs, self.kernels, self.bias)
        for i in range(len(self.hidden_units)):
            act_layer = self.activation_layers[i]
            dense = first if (i == 0 and first is not None) else \
                (lambda k, b, a, x=deep_input: ops.dense(x, k, b, a))
            if act_layer is None:
                fc = dense(self.kernels[i], self.bias[i], self.act_names[i])
            else:
                fc = dense(self.kernels[i], self.bias[i], None)
                if self.use_bn:
                    self.bn_layers[i]._maybe_build(fc.shape)
                    fc = self.bn_layers[i].call(fc, training=training)
                act_layer._maybe_build(fc.shape)
                fc = act_layer.call(fc, training=training)
            if self.dropout_rate and training:
                fc = self.dropout_layers[i].call(fc, training=training)
            deep_input = fc
        return deep_input

    def compute_output_shape(self, input_shape):
        if len(self.hidden_units) > 0:
            shape = tuple(input_shape[:-1]) + (self.hidden_units[-1],)
        else:
            shape = input_shape
        return tuple(shape)

    def get_config(self):
        config = {'activation': self.activation, 'hidden_units': self.hidden_units,
                  'l2_reg': self.l2_reg, 'use_bn': self.use_bn, 'dropout_rate': self.dropout_rate,
                  'output_activation': self.output_activation, 'seed': self.seed}
        base = Layer.get_config(self)
        return dict(list(base.items()) + list(config.items()))


class PredictionLayer(Layer):
    """deepctr/layers/core.py:226-267: + global_bias -> sigmoid (binary) -> reshape (-1, 1).
    During training the Model fuses this layer with the loss (b2ctr_predict_loss)."""

    def __init__(self, task='binary', use_bias=True, **kwargs):
        if task not in ["binary", "multiclass", "regression"]:
            raise ValueError("task must be binary,multiclass or regression")
        self.task = task
        self.use_bias = use_bias
        Layer.__init__(self, **kwargs)

    def build(self, input_shape):
        if self.use_bias:
            self.global_bias = self.add_weight(shape=(1,), initializer=Zeros(), name="global_bias")
        self.built = True

    def call(self, inputs, **kwargs):
        from .. import kernels as K
        # "multiclass" is, in the reference, exactly "no sigmoid" (core.py:250-257): bias, then reshape(-1, 1)
        lt = E.contiguous(inputs).reshape(-1)
        bias = self.global_bias.materialize() if self.use_bias else None
        task = L.TASK_BINARY if self.task == "binary" else L.TASK_REGRESSION
        pred, _, _, _ = K.predict_loss(lt, bias, None, task)
        return E.Var(pred.reshape(-1, 1))

    def compute_output_shape(self, input_shape):
        return (None, 1)

    def get_config(self):
        config = {'task': self.task, 'use_bias': self.use_bias}
        base = Layer.get_config(self)
        return dict(list(base.items()) + list(config.items()))


class LocalActivationUnit(Layer):
    """deepctr/layers/core.py:28-120: DIN's attention scorer.
    att_in = [q, k, q-k, q*k] -> DNN(hidden, act) -> . kernel + bias -> [B, T, 1]."""

    def __init__(self, hidden_units=(64, 32), activation='sigmoid', l2_reg=0, dropout_rate=0, use_bn=False,
                 seed=1024, **kwargs):
        self.hidden_units = hidden_units
        self.activation = activation
        self.l2_reg = l2_reg
        self.dropout_rate = dropout_rate
        self.use_bn = use_bn
        self.seed = seed
        Layer.__init__(self, **kwargs)
        self.supports_masking = True

    def build(self, input_shape):
        if not isinstance(input_shape, list) or len(input_shape) != 2:
            raise ValueError('A `LocalActivationUnit` layer should be called on a list of 2 inputs')
        if len(input_shape[0]) != 3 or len(input_shape[1]) != 3:
            raise ValueError("Unexpected inputs dimensions %d and %d, expect to be 3 dimensions" % (
                len(input_shape[0]), len(input_shape[1])))
        if input_shape[0][-1] != input_shape[1][-1] or input_shape[0][1] != 1:
            raise ValueError('A `LocalActivationUnit` layer requires '
                             'inputs of a two inputs with shape (None,1,embedding_size) and (None,T,embedding_size)'
                             'Got different shapes: %s,%s' % (input_shape[0], input_shape[1]))
        size = 4 * int(input_shape[0][-1]) if len(self.hidden_units) == 0 else self.hidden_units[-1]
        self.kernel = self.add_weight(shape=(size, 1), initializer=glorot_normal(seed=self.seed), name="kernel")
        self.bias = self.add_weight(shape=(1,), initializer=Zeros(), name="bias")
        self.dnn = self._track(DNN(self.hidden_units, self.activation, self.l2_reg, self.dropout_rate,
                                   self.use_bn, seed=self.seed, name=self.name + "/dnn"))
        self.dnn._maybe_build((input_shape[1][0], input_shape[1][1], 4 * int(input_shape[0][-1])))
        self.built = True

    def call(self, inputs, training=None, **kwargs):
        query, keys = inputs
        if len(self.hidden_units) > 0 and ops.din_att_fusable(query, keys, int(self.hidden_units[0])):
            # [q, k, q-k, q*k] is generated inside the first GEMM's producer: the [B,T,4E] tensor never exists
            att_out = self.dnn.call(None, training=training,
                                    first=lambda k, b, a: ops.din_att_first(query, keys, k, b, a))
        else:
            att_input = ops.din_att_input(query, keys)                   # [B,T,4E]   core.py:98-101
            att_out = self.dnn.call(att_input, training=training)        # core.py:103
        return ops.dense(att_out, self.kernel, self.bias, None)          # [B,T,1]    core.py:106

    def compute_output_shape(self, input_shape):
        return tuple(input_shape[1][:2]) + (1,)

    def compute_mask(self, inputs, mask=None):
        return mask

    def get_config(self):
        config = {'activation': self.activation, 'hidden_units': self.hidden_units,
                  'l2_reg': self.l2_reg, 'dropout_rate': self.dropout_rate, 'use_bn': self.use_bn,
                  'seed': self.seed}
        base = Layer.get_config(self)
        return dict(list(base.items()) + list(config.items()))


class RegulationModule(Layer):
    """EDCN's field-wise gate, deepctr/layers/core.py:270-321: [B, F, E] -> [B, F*E],
    y = x * softmax_f(g * (1 / tau)) with the weight g [1, F, 1].  As in the reference, ``self.tau`` holds 1 / tau and
    ``get_config`` returns it.  On its own the layer is one b2ctr_regulate launch in 'copy' mode; in EDCN the planner
    (inputs.RegulatePlan) serves two modules reading one tensor, and the bridge in front of them, with one launch."""

    def __init__(self, tau=1.0, **kwargs):
        if tau == 0:
            raise ValueError("RegulationModule tau can not be zero.")
        self.tau = 1.0 / tau
        Layer.__init__(self, **kwargs)

    def build(self, input_shape):
        self.field_size = int(input_shape[1])
        self.embedding_size = int(input_shape[2])
        self.g = self.add_weight(shape=(1, self.field_size, 1), initializer=Ones(), name=self.name + '_field_weight')
        self.built = True

    def call(self, inputs, **kwargs):
        if inputs.data.dim() != 3:
            raise ValueError("Unexpected inputs dimensions %d, expect to be 3 dimensions" % (inputs.data.dim()))
        _, (y,) = ops.regulate("copy", inputs, gates=[(self.g, self.tau)], want_u=False)
        return y

    def compute_output_shape(self, input_shape):
        return (None, self.field_size * self.embedding_size)

    def get_config(self):
        config = {'tau': self.tau}
        base = Layer.get_config(self)
        base.update(config)
        return base
