"""FLEN (Chen et al. 2019) - drop-in for the reference builder deepctr/models/flen.py:20-82.

The sparse embeddings are grouped by ``group_name``; FieldWiseBiInteraction takes one field-axis concatenation per
group, and its [B, E] output is concatenated with the DNN's output before the final Dense.  The planner
(inputs.FieldWisePlan) runs the layer in one b2ctr_field_wise_bi launch that reads every group's members in place
in the gather buffer, so the per-group concatenations are never written; its backward adds dx straight into the
gather buffer's gradient.

As in the reference, a single group raises the layer's ValueError when the model is built.  Deviation: embedding
dimensions that differ raise a ValueError naming both (the reference fails inside the concatenation)."""
from itertools import chain

from ..engine import Dense, Model
from ..feature_column import build_input_features, get_linear_logit, input_from_feature_columns
from ..layers.core import PredictionLayer, DNN
from ..layers.interaction import FieldWiseBiInteraction
from ..layers.utils import concat_func, add_func, combined_dnn_input


def FLEN(linear_feature_columns,
         dnn_feature_columns,
         dnn_hidden_units=(256, 128, 64),
         l2_reg_linear=0.00001,
         l2_reg_embedding=0.00001,
         l2_reg_dnn=0,
         seed=1024,
         dnn_dropout=0.0,
         dnn_activation='relu',
         dnn_use_bn=False,
         task='binary'):
    features = build_input_features(linear_feature_columns +
                                    dnn_feature_columns)

    inputs_list = list(features.values())

    group_embedding_dict, dense_value_list = input_from_feature_columns(
        features,
        dnn_feature_columns,
        l2_reg_embedding,
        seed,
        support_group=True)
    dims = sorted(set(int(e.shape[-1]) for v in group_embedding_dict.values() for e in v))
    if len(dims) > 1:
        raise ValueError("FLEN needs one embedding dimension for every field, got embedding dimensions %d and %d"
                         % (dims[0], dims[-1]))

    linear_logit = get_linear_logit(features,
                                    linear_feature_columns,
                                    seed=seed,
                                    prefix='linear',
                                    l2_reg=l2_reg_linear)

    fm_mf_out = FieldWiseBiInteraction(seed=seed)(
        [concat_func(v, axis=1) for k, v in group_embedding_dict.items()])

    dnn_input = combined_dnn_input(
        list(chain.from_iterable(group_embedding_dict.values())),
        dense_value_list)
    dnn_output = DNN(dnn_hidden_units, dnn_activation, l2_reg_dnn, dnn_dropout, dnn_use_bn, seed=seed)(dnn_input)

    dnn_logit = Dense(1, use_bias=False)(concat_func([fm_mf_out, dnn_output]))

    final_logit = add_func([linear_logit, dnn_logit])
    output = PredictionLayer(task)(final_logit)

    model = Model(inputs=inputs_list, outputs=output)
    return model
