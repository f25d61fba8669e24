"""AFM (Xiao et al. 2017) - drop-in for the reference builder deepctr/models/afm.py:19-61.
logit = first-order term + sum over the groups in `fm_group` of AFMLayer (or FM when use_attention=False).
The embeddings are looked up before the linear logit is built, as in the reference (layer and weight order)."""
from ..engine import Model
from ..feature_column import (DEFAULT_GROUP_NAME, build_input_features, get_linear_logit,
                              input_from_feature_columns)
from ..layers.core import PredictionLayer
from ..layers.interaction import AFMLayer, FM
from ..layers.utils import add_func, concat_func


def AFM(linear_feature_columns, dnn_feature_columns, fm_group=DEFAULT_GROUP_NAME, use_attention=True,
        attention_factor=8, l2_reg_linear=1e-5, l2_reg_embedding=1e-5, l2_reg_att=1e-5, afm_dropout=0, seed=1024,
        task='binary'):
    features = build_input_features(linear_feature_columns + dnn_feature_columns)
    inputs_list = list(features.values())
    group_embedding_dict, _ = input_from_feature_columns(features, dnn_feature_columns, l2_reg_embedding, seed,
                                                         support_dense=False, support_group=True)
    linear_logit = get_linear_logit(features, linear_feature_columns, seed=seed, prefix='linear',
                                    l2_reg=l2_reg_linear)
    # `k in fm_group` is a substring test when fm_group is the default string, as in the reference
    if use_attention:
        fm_logit = add_func([AFMLayer(attention_factor, l2_reg_att, afm_dropout, seed)(list(v))
                             for k, v in group_embedding_dict.items() if k in fm_group])
    else:
        fm_logit = add_func([FM()(concat_func(v, axis=1)) for k, v in group_embedding_dict.items() if k in fm_group])
    final_logit = add_func([linear_logit, fm_logit])
    return Model(inputs=inputs_list, outputs=PredictionLayer(task)(final_logit))
