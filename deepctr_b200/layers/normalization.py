"""BatchNormalization / Dropout used by DNN(use_bn, dropout_rate) (deepctr/layers/core.py:177-179), and the
reference's LayerNormalization (deepctr/layers/normalization.py:18-51) used by the Transformer layer of BST."""
from .. import ops
from ..engine import Layer, Zeros, Ones


class BatchNormalization(Layer):
    """tf.keras.layers.BatchNormalization defaults: momentum 0.99, epsilon 1e-3, gamma/beta trainable."""

    def __init__(self, axis=-1, momentum=0.99, epsilon=1e-3, center=True, scale=True, **kwargs):
        Layer.__init__(self, **kwargs)
        self.momentum, self.epsilon, self.center, self.scale = momentum, epsilon, center, scale

    def build(self, input_shape):
        n = int(input_shape[-1])
        self.gamma = self.add_weight("gamma", (n,), Ones()) if self.scale else None
        self.beta = self.add_weight("beta", (n,), Zeros()) if self.center else None
        self.moving_mean = self.add_weight("moving_mean", (n,), Zeros(), trainable=False)
        self.moving_variance = self.add_weight("moving_variance", (n,), Ones(), trainable=False)
        self.built = True

    def call(self, inputs, training=None, **kwargs):
        return ops.batchnorm(inputs, self.gamma, self.beta, self.moving_mean, self.moving_variance,
                             self.epsilon, bool(training), self.momentum)


class Dropout(Layer):
    def __init__(self, rate, seed=None, **kwargs):
        Layer.__init__(self, **kwargs)
        self.rate, self.seed = rate, seed
        self._calls = 0

    def next_seed(self):
        """Seed of this layer's next dropout mask (also drawn by the Transformer's fused attention dropout)."""
        self._calls += 1
        return (self.seed or 0) * 1000003 + self._calls

    def call(self, inputs, training=None, **kwargs):
        if not training or not self.rate:
            return inputs
        return ops.dropout(inputs, self.rate, self.next_seed())


class LayerNormalization(Layer):
    """(x - mean) / sqrt(var + eps) * gamma + beta over the last axis (deepctr/layers/normalization.py:18-51);
    gamma and beta are always created, ``scale`` / ``center`` only decide whether the call uses them."""

    def __init__(self, axis=-1, eps=1e-9, center=True, scale=True, **kwargs):
        if axis != -1:
            raise NotImplementedError("LayerNormalization over axis %r: only the last axis (-1) is supported" % (axis,))
        self.axis, self.eps, self.center, self.scale = axis, eps, center, scale
        Layer.__init__(self, **kwargs)

    def build(self, input_shape):
        self.gamma = self.add_weight(name='gamma', shape=tuple(input_shape[-1:]), initializer=Ones(), trainable=True)
        self.beta = self.add_weight(name='beta', shape=tuple(input_shape[-1:]), initializer=Zeros(), trainable=True)
        self.built = True

    def call(self, inputs, residual=None, **kwargs):
        """``residual``: normalise inputs + residual, the sum formed inside the kernel."""
        return ops.layernorm(inputs, self.gamma if self.scale else None, self.beta if self.center else None,
                             self.eps, b=residual)

    def compute_output_shape(self, input_shape):
        return input_shape

    def get_config(self):
        config = {'axis': self.axis, 'eps': self.eps, 'center': self.center, 'scale': self.scale}
        base = Layer.get_config(self)
        return dict(list(base.items()) + list(config.items()))
