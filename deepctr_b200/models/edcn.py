"""EDCN (Chen et al. 2021) - drop-in for the reference builder deepctr/models/edcn.py:21-103.

DCN plus information sharing: every layer is one CrossNet(1) and one DNN([F*E]); a BridgeModule joins their
outputs and two RegulationModules gate the bridge, per field, into the next layer's cross and deep inputs.  The
planner (inputs.RegulatePlan) serves the two gates of layer 0 with one launch over the gather buffer, and each inner
bridge with its two gates with one launch that never writes the bridge output.

As in the reference, the model's inputs are those of ``dnn_feature_columns`` only, so a linear column missing from
them raises KeyError, and dense features are rejected.  Deviations: a negative ``cross_num`` raises the reference's
ValueError (the reference fails with UnboundLocalError), and embedding dimensions that differ raise a ValueError
naming both (the reference fails inside the concatenation)."""
from ..engine import Concatenate, Dense, Model, Reshape
from ..feature_column import build_input_features, get_linear_logit, input_from_feature_columns
from ..layers.core import DNN, PredictionLayer, RegulationModule
from ..layers.interaction import BridgeModule, CrossNet
from ..layers.utils import add_func, concat_func


def EDCN(linear_feature_columns,
         dnn_feature_columns,
         cross_num=2,
         cross_parameterization='vector',
         bridge_type='concatenation',
         tau=1.0,
         l2_reg_linear=1e-5,
         l2_reg_embedding=1e-5,
         l2_reg_cross=1e-5,
         l2_reg_dnn=0,
         seed=1024,
         dnn_dropout=0,
         dnn_use_bn=False,
         dnn_activation='relu',
         task='binary'):
    if cross_num <= 0:
        raise ValueError("Cross layer num must > 0")

    print('EDCN brige type: ', bridge_type)

    features = build_input_features(dnn_feature_columns)
    inputs_list = list(features.values())

    linear_logit = get_linear_logit(features, linear_feature_columns, seed=seed, prefix='linear', l2_reg=l2_reg_linear)

    sparse_embedding_list, _ = input_from_feature_columns(
        features, dnn_feature_columns, l2_reg_embedding, seed, support_dense=False)
    dims = sorted(set(int(e.shape[-1]) for e in sparse_embedding_list))
    if len(dims) > 1:
        raise ValueError("EDCN needs one embedding dimension for every field, got embedding dimensions %d and %d"
                         % (dims[0], dims[-1]))

    emb_input = concat_func(sparse_embedding_list, axis=1)
    deep_in = RegulationModule(tau)(emb_input)
    cross_in = RegulationModule(tau)(emb_input)

    field_size = len(sparse_embedding_list)
    embedding_size = int(sparse_embedding_list[0].shape[-1])
    cross_dim = field_size * embedding_size

    for i in range(cross_num):
        cross_out = CrossNet(1, parameterization=cross_parameterization,
                             l2_reg=l2_reg_cross)(cross_in)
        deep_out = DNN([cross_dim], dnn_activation, l2_reg_dnn,
                       dnn_dropout, dnn_use_bn, seed=seed)(deep_in)
        print(cross_out, deep_out)
        bridge_out = BridgeModule(bridge_type)([cross_out, deep_out])
        if i + 1 < cross_num:
            bridge_out_list = Reshape([field_size, embedding_size])(bridge_out)
            deep_in = RegulationModule(tau)(bridge_out_list)
            cross_in = RegulationModule(tau)(bridge_out_list)

    stack_out = Concatenate()([cross_out, deep_out, bridge_out])
    final_logit = Dense(1, use_bias=False)(stack_out)

    final_logit = add_func([final_logit, linear_logit])
    output = PredictionLayer(task)(final_logit)

    model = Model(inputs=inputs_list, outputs=output)

    return model
