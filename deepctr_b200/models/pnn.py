"""PNN (Qu et al. 2016) - drop-in for the reference builder deepctr/models/pnn.py:18-71.
DNN input = [embeddings F*E || inner products P || outer products P || dense features], per use_inner / use_outter.

As in the reference, InnerProductLayer and OutterProductLayer are both created and called whatever the switches say;
a product that is not on the output path holds no weight in the model and launches nothing.  When the concatenation
reaches the first DNN layer only through combined_dnn_input, the products are written straight into the gather buffer
between the embeddings and the dense columns (inputs.EmbeddingPlanner._pnn_products), so the DNN input is a
zero-copy window of it."""
from ..engine import Dense, Flatten, Model, Reshape
from ..feature_column import build_input_features, input_from_feature_columns
from ..layers.core import DNN, PredictionLayer
from ..layers.interaction import InnerProductLayer, OutterProductLayer
from ..layers.utils import combined_dnn_input, concat_func


def PNN(dnn_feature_columns, dnn_hidden_units=(256, 128, 64), l2_reg_embedding=0.00001, l2_reg_dnn=0,
        seed=1024, dnn_dropout=0, dnn_activation='relu', use_inner=True, use_outter=False, kernel_type='mat',
        task='binary'):
    if kernel_type not in ['mat', 'vec', 'num']:
        raise ValueError("kernel_type must be mat,vec or num")
    features = build_input_features(dnn_feature_columns)
    inputs_list = list(features.values())
    sparse_embedding_list, dense_value_list = input_from_feature_columns(features, dnn_feature_columns,
                                                                         l2_reg_embedding, seed)
    inner_product = Flatten()(InnerProductLayer()(sparse_embedding_list))
    outter_product = OutterProductLayer(kernel_type)(sparse_embedding_list)
    linear_signal = Reshape([sum(int(x.shape[-1]) for x in sparse_embedding_list)])(
        concat_func(sparse_embedding_list))
    if use_inner and use_outter:
        deep_input = concat_func([linear_signal, inner_product, outter_product])
    elif use_inner:
        deep_input = concat_func([linear_signal, inner_product])
    elif use_outter:
        deep_input = concat_func([linear_signal, outter_product])
    else:
        deep_input = linear_signal
    dnn_input = combined_dnn_input([deep_input], dense_value_list)
    dnn_out = DNN(dnn_hidden_units, dnn_activation, l2_reg_dnn, dnn_dropout, False, seed=seed)(dnn_input)
    dnn_logit = Dense(1, use_bias=False)(dnn_out)
    output = PredictionLayer(task)(dnn_logit)
    return Model(inputs=inputs_list, outputs=output)
