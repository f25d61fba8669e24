"""CCPM (Liu et al. 2015) - drop-in for the reference builder deepctr/models/ccpm.py:21-82.

The embeddings of the sparse fields form a [B, n, E, 1] map; each layer is a Conv2D with a (width, 1) kernel and
tanh, then KMaxPooling along the fields; the flattened result feeds the DNN.  The planner (inputs.ConvStackPlan)
runs the whole stack in one b2ctr_conv_stack launch that reads the gather buffer in place and writes only the
flattened DNN input.

As in the reference, the model's inputs come from ``linear_feature_columns + dnn_feature_columns``, a DenseFeat in
``dnn_feature_columns`` raises ValueError (dense features in the linear columns only are legal), and the k of layer
i < l is max(1, int((1 - (i / l) ** (l - i)) * n)) with n the number of sparse embeddings, the last layer's 3, both
clamped to the rows they pool (ccpm.py:62-70).  Deviation: embedding dimensions that differ raise a ValueError
naming both (the reference fails inside the concatenation)."""
from .. import backend
from ..engine import Conv2D, Dense, Flatten, Lambda, Model
from ..feature_column import build_input_features, get_linear_logit, input_from_feature_columns
from ..layers.core import DNN, PredictionLayer
from ..layers.sequence import KMaxPooling
from ..layers.utils import add_func, concat_func


def ccpm_k(i, l, n):
    """k of conv layer i (1-based) of l over n sparse embeddings, before the clamp to the rows (ccpm.py:62)."""
    return max(1, int((1 - pow(i / l, l - i)) * n)) if i < l else 3


def CCPM(linear_feature_columns, dnn_feature_columns, conv_kernel_width=(6, 5), conv_filters=(4, 4),
         dnn_hidden_units=(128, 64), l2_reg_linear=1e-5, l2_reg_embedding=1e-5, l2_reg_dnn=0, dnn_dropout=0,
         seed=1024, task='binary'):
    if len(conv_kernel_width) != len(conv_filters):
        raise ValueError(
            "conv_kernel_width must have same element with conv_filters")

    features = build_input_features(
        linear_feature_columns + dnn_feature_columns)
    inputs_list = list(features.values())

    linear_logit = get_linear_logit(features, linear_feature_columns, seed=seed,
                                    l2_reg=l2_reg_linear)

    sparse_embedding_list, _ = input_from_feature_columns(features, dnn_feature_columns, l2_reg_embedding,
                                                          seed, support_dense=False)
    dims = sorted(set(int(e.shape[-1]) for e in sparse_embedding_list))
    if len(dims) > 1:
        raise ValueError("CCPM needs one embedding dimension for every field, got embedding dimensions %d and %d"
                         % (dims[0], dims[-1]))

    n = len(sparse_embedding_list)
    l = len(conv_filters)

    conv_input = concat_func(sparse_embedding_list, axis=1)
    pooling_result = Lambda(
        lambda x: backend.expand_dims(x, axis=3))(conv_input)

    for i in range(1, l + 1):
        filters = conv_filters[i - 1]
        width = conv_kernel_width[i - 1]
        k = ccpm_k(i, l, n)

        conv_result = Conv2D(filters=filters, kernel_size=(width, 1), strides=(1, 1), padding='same',
                             activation='tanh', use_bias=True, )(pooling_result)
        pooling_result = KMaxPooling(
            k=min(k, int(conv_result.shape[1])), axis=1)(conv_result)

    flatten_result = Flatten()(pooling_result)
    dnn_out = DNN(dnn_hidden_units, l2_reg=l2_reg_dnn, dropout_rate=dnn_dropout)(flatten_result)
    dnn_logit = Dense(1, use_bias=False)(
        dnn_out)

    final_logit = add_func([dnn_logit, linear_logit])

    output = PredictionLayer(task)(final_logit)
    model = Model(inputs=inputs_list, outputs=output)
    return model
