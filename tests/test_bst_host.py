"""CPU: the Transformer / PositionEncoding / LayerNormalization layers and the BST builder without a device -
argument checks and messages, weight names and order, initial tables, static shapes and configs."""
import numpy as np
import pytest

from deepctr_b200 import engine as E


def _build(layer, shapes):
    E.clear_session()
    ins = [E.Input(shape=s[1:], dtype="int32" if len(s) == 2 else "float32") for s in shapes]
    return layer(ins if len(ins) > 1 else ins[0])


def _transformer(**kw):
    from deepctr_b200.layers import Transformer
    E.clear_session()
    return Transformer(**kw)


def test_transformer_argument_checks():
    with pytest.raises(ValueError, match="head_num must be a int > 0"):
        _transformer(head_num=0)
    t = _transformer(att_embedding_size=3, head_num=2)
    with pytest.raises(ValueError, match=r"att_embedding_size \* head_num must equal the last dimension size of "
                                         r"inputs,got 3 \* 2 != 8"):
        t.build([(None, 5, 8), (None, 5, 8), (None, 1), (None, 1)])
    for kind in ("cos", "ln", "additive"):
        t = _transformer(att_embedding_size=4, head_num=2, attention_type=kind)
        with pytest.raises(NotImplementedError, match=kind):
            t.build([(None, 5, 8), (None, 5, 8), (None, 1), (None, 1)])
    t = _transformer(att_embedding_size=4, head_num=2)
    with pytest.raises(ValueError, match="T <= 128"):
        t.build([(None, 129, 8), (None, 129, 8), (None, 1), (None, 1)])
    t = _transformer(att_embedding_size=65, head_num=1)
    with pytest.raises(ValueError, match="att_embedding_size <= 64"):
        t.build([(None, 5, 65), (None, 5, 65), (None, 1), (None, 1)])


def test_layer_normalization_axis():
    from deepctr_b200.layers import LayerNormalization
    with pytest.raises(NotImplementedError):
        LayerNormalization(axis=1)
    ln = LayerNormalization()
    assert ln.get_config()["eps"] == 1e-9 and ln.get_config()["axis"] == -1


def test_transformer_weights_shapes_and_config():
    from deepctr_b200.layers import Transformer, custom_objects
    E.clear_session()
    q = E.Input(shape=(7, 8))
    ln = E.Input(shape=(1,), dtype="int32")
    t = Transformer(att_embedding_size=4, head_num=2, use_layer_norm=True, blinding=False, output_type=None)
    out = t([q, q, ln, ln])
    assert out.shape == (None, 7, 8)
    assert [w.name for w in t.weights] == [
        "transformer/query", "transformer/key", "transformer/value", "transformer/fw1", "transformer/fw2",
        "transformer/ln/gamma", "transformer/ln/beta", "transformer/query_pe/lookup_table",
        "transformer/key_pe/lookup_table"]
    assert t.weights[3].shape == (8, 32) and t.weights[4].shape == (32, 8)
    # the nested layers took the next automatic names of their classes
    from deepctr_b200.layers import Dropout, LayerNormalization, PositionEncoding
    assert Dropout(0.1).name == "dropout_1"
    assert LayerNormalization().name == "layer_normalization_1"
    assert PositionEncoding().name == "position_encoding_2"
    cfg = t.get_config()
    for k in ("att_embedding_size", "head_num", "dropout_rate", "use_res", "use_positional_encoding",
              "use_feed_forward", "use_layer_norm", "seed", "supports_masking", "blinding", "attention_type",
              "output_type"):
        assert k in cfg
    for name in ("Transformer", "PositionEncoding", "LayerNormalization"):
        assert name in custom_objects
    E.clear_session()
    pooled = Transformer(att_embedding_size=1, head_num=8, output_type="sum")([q, q, ln, ln])
    assert pooled.shape == (None, 1, 8)


def test_position_encoding_table():
    from deepctr_b200.layers import PositionEncoding
    for zero_pad in (False, True):
        E.clear_session()
        pe = PositionEncoding(zero_pad=zero_pad)
        pe.build((None, 6, 8))
        tab = pe.lookup_table.value()
        pos = np.arange(6)[:, None] / np.power(10000, 2.0 * (np.arange(8) // 2) / 8)[None, :]
        want = np.where(np.arange(8) % 2 == 0, np.sin(pos), np.cos(pos))
        if zero_pad:
            want[0] = 0
        np.testing.assert_allclose(tab, want.astype(np.float32), rtol=1e-6, atol=1e-7)
    E.clear_session()
    pe = PositionEncoding(pos_embedding_trainable=False)
    pe.build((None, 6, 8))
    assert not pe.lookup_table.trainable


def _cols(T=4):
    from deepctr_b200.feature_column import SparseFeat, VarLenSparseFeat, DenseFeat
    cols = [SparseFeat('user', 3, embedding_dim=8), SparseFeat('gender', 2, embedding_dim=8),
            SparseFeat('item_id', 4, embedding_dim=8), SparseFeat('cate_id', 3, embedding_dim=8),
            DenseFeat('pay_score', 1)]
    cols += [VarLenSparseFeat(SparseFeat('hist_item_id', 4, embedding_dim=8, embedding_name='item_id'), maxlen=T,
                              length_name="seq_length"),
             VarLenSparseFeat(SparseFeat('hist_cate_id', 3, embedding_dim=8, embedding_name='cate_id'), maxlen=T,
                              length_name="seq_length")]
    return cols


def test_bst_builder_weights_and_graph():
    from deepctr_b200 import models as M
    E.clear_session()
    model = M.BST(_cols(), ['item_id', 'cate_id'], att_head_num=4)
    names = [w.name for w in model.weights]
    assert names[:4] == ["sparse_emb_user/embeddings", "sparse_emb_gender/embeddings", "sparse_emb_item_id/embeddings",
                         "sparse_emb_cate_id/embeddings"]
    assert names[4:13] == ["transformer/query", "transformer/key", "transformer/value", "transformer/fw1",
                           "transformer/fw2", "transformer/ln/gamma", "transformer/ln/beta",
                           "transformer/query_pe/lookup_table", "transformer/key_pe/lookup_table"]
    assert model.get_layer("transformer").att_embedding_size == 4
    assert names[-1] == "prediction_layer/global_bias" and names[-2] == "dense/kernel"
    assert any(n.startswith("attention_sequence_pooling_layer/local_activation_unit/dnn/kernel0") for n in names)
    t = model.get_layer("transformer")
    assert (t.blinding, t.use_layer_norm, t.output_type, t.supports_masking) == (False, True, None, False)
    att = model.get_layer("attention_sequence_pooling_layer")
    assert (att.att_hidden_units, att.weight_normalization, att.supports_masking) == ((64, 16), True, False)


def test_bst_two_layers_and_errors():
    from deepctr_b200 import models as M
    E.clear_session()
    model = M.BST(_cols(), ['item_id', 'cate_id'], transformer_num=2, att_head_num=2, dnn_dropout=0.5)
    assert model.get_layer("transformer_1").dropout_rate == 0.5
    E.clear_session()
    with pytest.raises(ValueError, match="must equal the last dimension"):
        M.BST(_cols(), ['item_id', 'cate_id'], att_head_num=3)
    E.clear_session()
    with pytest.raises(ValueError, match="T <= 128"):
        M.BST(_cols(T=130), ['item_id', 'cate_id'], att_head_num=4)


def test_transformer_rejects_keys_of_another_shape():
    t = _transformer(att_embedding_size=4, head_num=2)
    with pytest.raises(ValueError, match="same shape"):
        t.build([(None, 7, 8), (None, 5, 8), (None, 1), (None, 1)])


def test_reference_builders_call_get_shape_as_list():
    E.clear_session()
    t = E.Input(shape=(4, 12))
    assert t.get_shape().as_list() == [None, 4, 12] and t.get_shape() == (None, 4, 12)
