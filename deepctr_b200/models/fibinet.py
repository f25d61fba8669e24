"""FiBiNET (Huang et al. 2019) - drop-in for the reference builder deepctr/models/fibinet.py:19-66.
logit = first-order term + DNN tower over [Bilinear(SENET(embeddings)) || Bilinear(embeddings) || dense features].
Both bilinear layers write their pairs into the DNN input where their Concat runs (inputs._bilinear_into_dnn_input)."""
from ..engine import Dense, Flatten
from ..layers.core import DNN
from ..layers.interaction import BilinearInteraction, SENETLayer
from ..layers.utils import combined_dnn_input, concat_func
from ._tower import Tower, total


def FiBiNET(linear_feature_columns, dnn_feature_columns, bilinear_type='interaction', reduction_ratio=3,
            dnn_hidden_units=(256, 128, 64), l2_reg_linear=1e-5, l2_reg_embedding=1e-5, l2_reg_dnn=0, seed=1024,
            dnn_dropout=0, dnn_activation='relu', task='binary'):
    t = Tower(linear_feature_columns + dnn_feature_columns, linear_feature_columns, dnn_feature_columns, seed,
              l2_reg_linear, l2_reg_embedding)
    senet_embedding_list = SENETLayer(reduction_ratio, seed)(t.embeddings)
    senet_bilinear_out = BilinearInteraction(bilinear_type=bilinear_type, seed=seed)(senet_embedding_list)
    bilinear_out = BilinearInteraction(bilinear_type=bilinear_type, seed=seed)(t.embeddings)
    dnn_input = combined_dnn_input([Flatten()(concat_func([senet_bilinear_out, bilinear_out]))], t.dense_values)
    dnn_out = DNN(dnn_hidden_units, dnn_activation, l2_reg_dnn, dnn_dropout, False, seed=seed)(dnn_input)
    dnn_logit = Dense(1, use_bias=False)(dnn_out)
    return t.finish(total([t.linear_logit, dnn_logit]), task)
