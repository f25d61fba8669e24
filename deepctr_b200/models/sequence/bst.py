"""Behavior Sequence Transformer (Chen et al. 2019) - drop-in for the reference builder
deepctr/models/sequence/bst.py:21-107.

The inputs are DIN's: the behaviour sequences are the VarLen columns called "hist_" + name, sharing their table with
the query column, and "seq_length" holds their lengths.  The sequence goes through ``transformer_num`` Transformer
layers (fused masked attention + LayerNormalization kernels), is pooled by DIN's attention unit against the query
and joins the other embeddings in front of the DNN tower."""
from ...engine import Dense, Flatten, Model
from ...feature_column import DenseFeat, SparseFeat, VarLenSparseFeat, build_input_features
from ... import inputs as I
from ...layers.core import DNN, PredictionLayer
from ...layers.sequence import AttentionSequencePoolingLayer, Transformer
from ...layers.utils import combined_dnn_input, concat_func


def BST(dnn_feature_columns, history_feature_list, transformer_num=1, att_head_num=8,
        use_bn=False, dnn_hidden_units=(256, 128, 64), dnn_activation='relu', l2_reg_dnn=0,
        l2_reg_embedding=1e-6, dnn_dropout=0.0, seed=1024, task='binary'):
    features = build_input_features(dnn_feature_columns)
    inputs_list = list(features.values())
    user_behavior_length = features["seq_length"]

    cols = dnn_feature_columns or []
    sparse_feature_columns = [c for c in cols if isinstance(c, SparseFeat)]
    dense_feature_columns = [c for c in cols if isinstance(c, DenseFeat)]
    varlen_sparse_feature_columns = [c for c in cols if isinstance(c, VarLenSparseFeat)]
    history_fc_names = ["hist_" + x for x in history_feature_list]
    history_feature_columns = [c for c in varlen_sparse_feature_columns if c.name in history_fc_names]
    sparse_varlen_feature_columns = [c for c in varlen_sparse_feature_columns if c.name not in history_fc_names]

    embedding_dict = I.create_embedding_matrix(dnn_feature_columns, l2_reg_embedding, seed, prefix="",
                                               seq_mask_zero=True)
    query_emb_list = I.embedding_lookup(embedding_dict, features, sparse_feature_columns,
                                        return_feat_list=history_feature_list, to_list=True)
    hist_emb_list = I.embedding_lookup(embedding_dict, features, history_feature_columns,
                                       return_feat_list=history_fc_names, to_list=True)
    dnn_input_emb_list = I.embedding_lookup(embedding_dict, features, sparse_feature_columns,
                                            mask_feat_list=history_feature_list, to_list=True)
    dense_value_list = I.get_dense_input(features, dense_feature_columns)
    sequence_embed_dict = I.varlen_embedding_lookup(embedding_dict, features, sparse_varlen_feature_columns)
    sequence_embed_list = I.get_varlen_pooling_list(sequence_embed_dict, features, sparse_varlen_feature_columns,
                                                    to_list=True)

    dnn_input_emb_list += sequence_embed_list
    query_emb = concat_func(query_emb_list)
    deep_input_emb = concat_func(dnn_input_emb_list)
    hist_emb = concat_func(hist_emb_list)

    transformer_output = hist_emb
    for _ in range(transformer_num):
        att_embedding_size = transformer_output.get_shape().as_list()[-1] // att_head_num
        transformer_layer = Transformer(att_embedding_size=att_embedding_size, head_num=att_head_num,
                                        dropout_rate=dnn_dropout, use_positional_encoding=True, use_res=True,
                                        use_feed_forward=True, use_layer_norm=True, blinding=False, seed=seed,
                                        supports_masking=False, output_type=None)
        transformer_output = transformer_layer([transformer_output, transformer_output,
                                                user_behavior_length, user_behavior_length])

    attn_output = AttentionSequencePoolingLayer(att_hidden_units=(64, 16), weight_normalization=True,
                                                supports_masking=False)([query_emb, transformer_output,
                                                                         user_behavior_length])
    deep_input_emb = concat_func([deep_input_emb, attn_output], axis=-1)
    deep_input_emb = Flatten()(deep_input_emb)

    dnn_input = combined_dnn_input([deep_input_emb], dense_value_list)
    output = DNN(dnn_hidden_units, dnn_activation, l2_reg_dnn, dnn_dropout, use_bn, seed=seed)(dnn_input)
    final_logit = Dense(1, use_bias=False)(output)
    output = PredictionLayer(task)(final_logit)
    return Model(inputs=inputs_list, outputs=output)
