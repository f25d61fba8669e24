"""DIFM (Lu et al. 2020) - drop-in for the reference builder deepctr/models/difm.py:20-82.
The field weights are m = Dense(F)(Flatten(InteractingLayer(x))) + Dense(F)(DNN(x)) (no softmax: unbounded, possibly
negative); the rest is IFM's: logit = linear(m) + FM(m ⊙ x), with the refined FM input never written.

InteractingLayer's limit applies: F * att_embedding_size * att_head_num <= 3072, so F <= 48 at the defaults (8, 8);
beyond it the layer raises ValueError when the model is built."""
from ..engine import Dense, Flatten
from ..layers.interaction import InteractingLayer
from ..layers.utils import add_func, combined_dnn_input
from .ifm import input_aware_tower, refined_fm_logit


def DIFM(linear_feature_columns, dnn_feature_columns,
         att_embedding_size=8, att_head_num=8, att_res=True, dnn_hidden_units=(256, 128, 64),
         l2_reg_linear=0.00001, l2_reg_embedding=0.00001, l2_reg_dnn=0, seed=1024, dnn_dropout=0,
         dnn_activation='relu', dnn_use_bn=False, task='binary'):
    t, nfield = input_aware_tower(linear_feature_columns, dnn_feature_columns, dnn_hidden_units, l2_reg_linear,
                                  l2_reg_embedding, seed)
    att_out = InteractingLayer(att_embedding_size, att_head_num, att_res, scaling=True)(t.field_matrix())
    m_vec = Dense(nfield, use_bias=False)(Flatten()(att_out))
    dnn_output = t.mlp(dnn_hidden_units, dnn_activation, l2_reg_dnn, dnn_dropout, dnn_use_bn,
                       inputs=combined_dnn_input(t.embeddings, []))
    m_bit = Dense(nfield, use_bias=False)(dnn_output)
    input_aware_factor = add_func([m_vec, m_bit])
    return refined_fm_logit(t, input_aware_factor, task)
