"""Host mirror of deepctr/layers/activation.py: Dice (:28-72) and activation_layer (:75-85)."""
from .. import ops
from ..engine import Layer, Zeros

_FUSABLE = ("relu", "sigmoid", "tanh", "linear", None)


def fusable_activation(name):
    """True when the activation can ride in the GEMM epilogue (b2ctr_gemm act codes)."""
    return name in _FUSABLE


class Activation(Layer):
    """tf.keras.layers.Activation for the string activations the reference uses.  'softmax' (the output activation of
    BridgeModule's attention DNNs) normalises the last axis of a 2-D tensor on b2ctr_softmax_rows; it cannot ride in
    a GEMM epilogue."""

    def __init__(self, activation, **kwargs):
        Layer.__init__(self, **kwargs)
        if not fusable_activation(activation) and activation != "softmax":
            raise ValueError("unsupported activation %r (relu, sigmoid, tanh, linear, dice)" % (activation,))
        self.activation = activation

    def call(self, inputs, **kwargs):
        if self.activation == "softmax":
            return ops.softmax(inputs)
        return ops.activation(inputs, self.activation)

    def get_config(self):
        c = Layer.get_config(self)
        c.update(activation=self.activation)
        return c


class Dice(Layer):
    """Data Adaptive Activation Function of DIN, deepctr/layers/activation.py:28-72:
    p = sigmoid(BN_{center=False, scale=False, eps}(x));  y = alpha * (1 - p) * x + p * x.
    Training uses batch statistics over all leading axes and updates the moving statistics with
    Keras' momentum 0.99; inference uses the moving statistics."""

    def __init__(self, axis=-1, epsilon=1e-9, **kwargs):
        self.axis = axis
        self.epsilon = epsilon
        Layer.__init__(self, **kwargs)

    def build(self, input_shape):
        from ..engine import Ones
        n = int(input_shape[-1])
        self.alphas = self.add_weight(shape=(n,), initializer=Zeros(), name='dice_alpha')
        self.moving_mean = self.add_weight(shape=(n,), initializer=Zeros(), name='bn/moving_mean',
                                           trainable=False)
        self.moving_variance = self.add_weight(shape=(n,), initializer=Ones(), name='bn/moving_variance',
                                               trainable=False)
        self.built = True

    def call(self, inputs, training=None, **kwargs):
        return ops.dice(inputs, self.alphas, self.moving_mean, self.moving_variance, self.epsilon,
                        bool(training), momentum=0.99)

    def compute_output_shape(self, input_shape):
        return input_shape

    def get_config(self):
        config = {'axis': self.axis, 'epsilon': self.epsilon}
        base = Layer.get_config(self)
        return dict(list(base.items()) + list(config.items()))


def activation_layer(activation, name=None):
    """deepctr/layers/activation.py:75-85."""
    if activation in ("dice", "Dice"):
        act_layer = Dice(name=name)
    elif isinstance(activation, str) or activation is None:
        act_layer = Activation(activation, name=name)
    elif isinstance(activation, type) and issubclass(activation, Layer):
        act_layer = activation()
    else:
        raise ValueError(
            "Invalid activation,found %s.You should use a str or a Activation Layer Class." % (activation))
    return act_layer
