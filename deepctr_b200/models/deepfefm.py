"""DeepFEFM (Pande 2020) - drop-in for the reference builder deepctr/models/deepfefm.py:23-106, with all of its
ablation switches.  FEFMLayer runs over DEFAULT_GROUP_NAME only; its P pair scores feed the DNN behind the
embeddings and the dense features, and their sum is the FEFM logit.

As in the reference, a DNN and a Dense(1) are created even when dnn_hidden_units is empty; they are not on the
output path then, so the model does not hold them (the names they took stay taken)."""
from ..engine import Dense, Lambda
from ..feature_column import DEFAULT_GROUP_NAME
from ..layers.core import DNN
from ..layers.interaction import FEFMLayer
from ..layers.utils import add_func, combined_dnn_input, concat_func, reduce_sum
from ._tower import Tower


def DeepFEFM(linear_feature_columns, dnn_feature_columns, use_fefm=True,
             dnn_hidden_units=(256, 128, 64), l2_reg_linear=0.00001, l2_reg_embedding_feat=0.00001,
             l2_reg_embedding_field=0.00001, l2_reg_dnn=0, seed=1024, dnn_dropout=0.0,
             exclude_feature_embed_in_dnn=False,
             use_linear=True, use_fefm_embed_in_dnn=True, dnn_activation='relu', dnn_use_bn=False, task='binary'):
    t = Tower(linear_feature_columns + dnn_feature_columns, linear_feature_columns, dnn_feature_columns, seed,
              l2_reg_linear, l2_reg_embedding_feat, grouped=True)
    fefm_interaction_embedding = concat_func([FEFMLayer(regularizer=l2_reg_embedding_field)(concat_func(v, axis=1))
                                              for k, v in t.groups.items() if k in [DEFAULT_GROUP_NAME]], axis=1)
    dnn_input = combined_dnn_input(t.embeddings, t.dense_values)
    if use_fefm_embed_in_dnn:
        if exclude_feature_embed_in_dnn:
            dnn_input = fefm_interaction_embedding
        else:
            dnn_input = concat_func([dnn_input, fefm_interaction_embedding], axis=1)
    dnn_out = DNN(dnn_hidden_units, dnn_activation, l2_reg_dnn, dnn_dropout, dnn_use_bn, seed=seed)(dnn_input)
    dnn_logit = Dense(1, use_bias=False, )(dnn_out)
    fefm_logit = Lambda(lambda x: reduce_sum(x, axis=1, keep_dims=True))(fefm_interaction_embedding)

    deep = len(dnn_hidden_units) > 0
    if not deep and not use_fefm and use_linear:
        final_logit = t.linear_logit
    elif not deep and use_fefm and use_linear:
        final_logit = add_func([t.linear_logit, fefm_logit])
    elif deep and not use_fefm and use_linear:
        final_logit = add_func([t.linear_logit, dnn_logit])
    elif deep and use_fefm and use_linear:
        final_logit = add_func([t.linear_logit, fefm_logit, dnn_logit])
    elif not deep and use_fefm and not use_linear:
        final_logit = fefm_logit
    elif deep and not use_fefm and not use_linear:
        final_logit = dnn_logit
    elif deep and use_fefm and not use_linear:
        final_logit = add_func([fefm_logit, dnn_logit])
    else:
        raise NotImplementedError
    return t.finish(final_logit, task)
