"""ONN / NFFM (Yang et al. 2019) - drop-in for the reference builder deepctr/models/onn.py:32-118.

Field-aware embeddings: every field a has one table ``sparse_emb_<a>_<b>`` per partner field b, and pair (i, j)
multiplies field i's row from its table for j with field j's row from its table for i.  The reference's dict
comprehension also declares the diagonal tables ``sparse_emb_<a>_<a>`` but never calls them, so Keras never builds
them; here they are not created at all.  The F(F-1) lookups, the P multiplies and the optional K.sum are served by
one field-aware product kernel (inputs.FieldAwarePlan), and concat_func + Flatten of the P products is a zero-copy
view of its output."""
import itertools

from .. import backend as K
from ..engine import Dense, Flatten, Lambda, Model, l2, multiply
from ..feature_column import SparseFeat, VarLenSparseFeat, build_input_features, get_linear_logit
from ..inputs import Embedding, get_dense_input, MAX_FFM_FIELDS, MAX_FFM_DIM
from ..layers.core import DNN, PredictionLayer
from ..layers.normalization import BatchNormalization
from ..layers.sequence import SequencePoolingLayer
from ..layers.utils import Hash, NoMask, add_func, combined_dnn_input, concat_func


def ONN(linear_feature_columns, dnn_feature_columns, dnn_hidden_units=(256, 128, 64),
        l2_reg_embedding=1e-5, l2_reg_linear=1e-5, l2_reg_dnn=0, dnn_dropout=0,
        seed=1024, use_bn=True, reduce_sum=False, task='binary',
        ):
    features = build_input_features(linear_feature_columns + dnn_feature_columns)
    inputs_list = list(features.values())
    linear_logit = get_linear_logit(features, linear_feature_columns, seed=seed, prefix='linear',
                                    l2_reg=l2_reg_linear)

    sparse_feature_columns = list(
        filter(lambda x: isinstance(x, SparseFeat), dnn_feature_columns)) if dnn_feature_columns else []
    varlen_sparse_feature_columns = list(
        filter(lambda x: isinstance(x, VarLenSparseFeat), dnn_feature_columns)) if dnn_feature_columns else []
    fields = sparse_feature_columns + varlen_sparse_feature_columns
    if not 2 <= len(fields) <= MAX_FFM_FIELDS:
        raise ValueError("ONN needs between 2 and %d sparse fields, got %d" % (MAX_FFM_FIELDS, len(fields)))
    for fc in fields:
        if fc.embedding_dim > MAX_FFM_DIM:
            raise ValueError("ONN supports embedding_dim <= %d, feature %r has %d"
                             % (MAX_FFM_DIM, fc.name, fc.embedding_dim))

    # the tables, keyed like the reference's dict (embedding_name -> embedding_name) and created at their first
    # call; onn.py's feature_embedding indexes them by fc.name, so a column whose embedding_name differs from its
    # name raises KeyError as it does there
    declared = {fc_j.embedding_name: {fc_i.embedding_name: fc_j for fc_i in fields} for fc_j in fields}
    tables = {}

    def table(fc_i, fc_j):
        owner = declared[fc_i.name][fc_j.name]
        key = (owner.embedding_name, fc_j.name)
        if key not in tables:
            tables[key] = Embedding(owner.vocabulary_size, owner.embedding_dim,
                                    embeddings_initializer=owner.embeddings_initializer,
                                    embeddings_regularizer=l2(l2_reg_embedding),
                                    mask_zero=isinstance(owner, VarLenSparseFeat),
                                    name='sparse_emb_' + str(owner.embedding_name) + '_' + fc_j.name)
        return tables[key]

    def feature_embedding(fc_i, fc_j, input_feature):
        fc_i_embedding = table(fc_i, fc_j)(input_feature)
        if isinstance(fc_i, SparseFeat):
            return NoMask()(fc_i_embedding)
        return SequencePoolingLayer(fc_i.combiner, supports_masking=True)(fc_i_embedding)

    dense_value_list = get_dense_input(features, dnn_feature_columns)

    embed_list = []
    for fc_i, fc_j in itertools.combinations(fields, 2):
        i_input = features[fc_i.name]
        if fc_i.use_hash:
            i_input = Hash(fc_i.vocabulary_size)(i_input)
        j_input = features[fc_j.name]
        if fc_j.use_hash:
            j_input = Hash(fc_j.vocabulary_size)(j_input)

        fc_i_embedding = feature_embedding(fc_i, fc_j, i_input)
        fc_j_embedding = feature_embedding(fc_j, fc_i, j_input)

        element_wise_prod = multiply([fc_i_embedding, fc_j_embedding])
        if reduce_sum:
            element_wise_prod = Lambda(lambda element_wise_prod: K.sum(
                element_wise_prod, axis=-1))(element_wise_prod)
        embed_list.append(element_wise_prod)

    ffm_out = Flatten()(concat_func(embed_list, axis=1))
    if use_bn:
        ffm_out = BatchNormalization()(ffm_out)
    dnn_input = combined_dnn_input([ffm_out], dense_value_list)
    dnn_out = DNN(dnn_hidden_units, l2_reg=l2_reg_dnn, dropout_rate=dnn_dropout)(dnn_input)
    dnn_logit = Dense(1, use_bias=False)(dnn_out)

    final_logit = add_func([dnn_logit, linear_logit])

    output = PredictionLayer(task)(final_logit)

    model = Model(inputs=inputs_list, outputs=output)
    return model
