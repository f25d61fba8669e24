"""NFM (He & Chua 2017) - drop-in for the reference builder deepctr/models/nfm.py:18-61.
logit = first-order term + DNN tower over [Bi-Interaction pooling of the embeddings || dense features]."""
from ..engine import Dense
from ..layers.core import DNN
from ..layers.interaction import BiInteractionPooling
from ..layers.normalization import Dropout
from ..layers.utils import combined_dnn_input
from ._tower import Tower, total


def NFM(linear_feature_columns, dnn_feature_columns, dnn_hidden_units=(256, 128, 64),
        l2_reg_embedding=1e-5, l2_reg_linear=1e-5, l2_reg_dnn=0, seed=1024, bi_dropout=0,
        dnn_dropout=0, dnn_activation='relu', task='binary'):
    t = Tower(linear_feature_columns + dnn_feature_columns, linear_feature_columns, dnn_feature_columns, seed,
              l2_reg_linear, l2_reg_embedding)
    bi_out = BiInteractionPooling()(t.field_matrix())
    if bi_dropout:
        bi_out = Dropout(bi_dropout)(bi_out, training=None)
    dnn_input = combined_dnn_input([bi_out], t.dense_values)
    dnn_output = DNN(dnn_hidden_units, dnn_activation, l2_reg_dnn, dnn_dropout, False, seed=seed)(dnn_input)
    dnn_logit = Dense(1, use_bias=False)(dnn_output)
    return t.finish(total([t.linear_logit, dnn_logit]), task)
