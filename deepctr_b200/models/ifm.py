"""IFM (Yu et al. 2019) - drop-in for the reference builder deepctr/models/ifm.py:21-74.
A DNN over the embeddings gives per-sample field weights m = F * softmax(Dense(F)(DNN(x))); they reweight the sparse
lookups of the first-order term and the FM input: logit = linear(m) + FM(m ⊙ x).  The refined FM input is never
written: FM receives it as its two factors and runs the field-weighted FM kernel (ops.scale_fields / ops.fm)."""
from .. import ops
from ..engine import Dense, Lambda
from ..feature_column import SparseFeat, VarLenSparseFeat
from ..layers.interaction import FM
from ..layers.utils import add_func, combined_dnn_input
from ._tower import Tower


def input_aware_tower(linear_feature_columns, dnn_feature_columns, dnn_hidden_units, l2_reg_linear, l2_reg_embedding,
                      seed):
    """The opening both input-aware builders share (ifm.py:40-57, difm.py:43-57): the checks, the inputs and the
    embeddings (the linear logit is built later, from the field weights), and F, the number of sparse and varlen
    columns among the DNN columns."""
    if not len(dnn_hidden_units) > 0:
        raise ValueError("dnn_hidden_units is null!")
    t = Tower(linear_feature_columns + dnn_feature_columns, linear_feature_columns, dnn_feature_columns, seed,
              l2_reg_linear, l2_reg_embedding, defer_linear=True)
    nfield = len([c for c in dnn_feature_columns if isinstance(c, (SparseFeat, VarLenSparseFeat))])
    if not len(t.embeddings) > 0:
        raise ValueError("there are no sparse features")
    return t, nfield


def refined_fm_logit(t, input_aware_factor, task):
    """linear(m) + FM(m ⊙ x) and the prediction head (ifm.py:62-74, difm.py:70-82)."""
    linear_logit = t.linear(input_aware_factor)
    refined_fm_input = Lambda(lambda x: ops.scale_fields(x[0], x[1]))([t.field_matrix(), input_aware_factor])
    fm_logit = FM()(refined_fm_input)
    return t.finish(add_func([linear_logit, fm_logit]), task)


def IFM(linear_feature_columns, dnn_feature_columns, dnn_hidden_units=(256, 128, 64),
        l2_reg_linear=0.00001, l2_reg_embedding=0.00001, l2_reg_dnn=0, seed=1024, dnn_dropout=0,
        dnn_activation='relu', dnn_use_bn=False, task='binary'):
    t, nfield = input_aware_tower(linear_feature_columns, dnn_feature_columns, dnn_hidden_units, l2_reg_linear,
                                  l2_reg_embedding, seed)
    dnn_output = t.mlp(dnn_hidden_units, dnn_activation, l2_reg_dnn, dnn_dropout, dnn_use_bn,
                       inputs=combined_dnn_input(t.embeddings, []))
    dnn_output = Dense(nfield, use_bias=False)(dnn_output)
    input_aware_factor = Lambda(lambda x: ops.softmax(x, dim=1, scale=x.shape[-1]))(dnn_output)
    return refined_fm_logit(t, input_aware_factor, task)
