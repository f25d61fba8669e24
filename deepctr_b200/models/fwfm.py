"""FwFM (Pan et al. 2018) - drop-in for the reference builder deepctr/models/fwfm.py:23-76.
logit = first-order term + sum over the groups in `fm_group` of FwFMLayer (+ a DNN tower over the embeddings and
the dense features when dnn_hidden_units is not empty)."""
from ..engine import Dense
from ..feature_column import DEFAULT_GROUP_NAME
from ..layers.core import DNN
from ..layers.interaction import FwFMLayer
from ..layers.utils import add_func, combined_dnn_input, concat_func
from ._tower import Tower


def FwFM(linear_feature_columns, dnn_feature_columns, fm_group=(DEFAULT_GROUP_NAME,), dnn_hidden_units=(256, 128, 64),
         l2_reg_linear=0.00001, l2_reg_embedding=0.00001, l2_reg_field_strength=0.00001, l2_reg_dnn=0,
         seed=1024, dnn_dropout=0, dnn_activation='relu', dnn_use_bn=False, task='binary'):
    t = Tower(linear_feature_columns + dnn_feature_columns, linear_feature_columns, dnn_feature_columns, seed,
              l2_reg_linear, l2_reg_embedding, grouped=True)
    fwfm_logit = add_func([FwFMLayer(num_fields=len(v), regularizer=l2_reg_field_strength)(concat_func(v, axis=1))
                           for k, v in t.groups.items() if k in fm_group])
    final_logit_components = [t.linear_logit, fwfm_logit]
    if dnn_hidden_units:
        dnn_input = combined_dnn_input(t.embeddings, t.dense_values)
        dnn_output = DNN(dnn_hidden_units, dnn_activation, l2_reg_dnn, dnn_dropout, dnn_use_bn, seed=seed)(dnn_input)
        final_logit_components.append(Dense(1, use_bias=False)(dnn_output))
    return t.finish(add_func(final_logit_components), task)
