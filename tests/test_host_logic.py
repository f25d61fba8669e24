"""CPU: host-side mirror of the reference interface - feature columns, graph construction for the five
builders, shapes, weight names, planner layout, build-time errors.  No kernels are launched."""
import numpy as np
import pytest

from deepctr_b200.feature_column import (SparseFeat, VarLenSparseFeat, DenseFeat, get_feature_names,
                                         build_input_features, input_from_feature_columns, DEFAULT_GROUP_NAME)
from deepctr_b200.models import DeepFM, xDeepFM, DCN, AutoInt, DIN


def _criteo(n_sparse=4, n_dense=3, dim=8):
    return [SparseFeat("C%d" % i, 10 + i, dim) for i in range(n_sparse)] + \
           [DenseFeat("I%d" % i, 1) for i in range(n_dense)]


def test_feature_column_defaults_follow_reference():
    # deepctr/feature_column.py:34-57
    s = SparseFeat("a", 1000)
    assert (s.embedding_dim, s.use_hash, s.dtype, s.embedding_name, s.group_name, s.trainable) == \
           (4, False, "int32", "a", DEFAULT_GROUP_NAME, True)
    assert s.embeddings_initializer.stddev == 0.0001 and s.embeddings_initializer.seed == 2020
    assert SparseFeat("b", 10000, "auto").embedding_dim == 6 * int(pow(10000, 0.25))       # :44-45
    v = VarLenSparseFeat(SparseFeat("h", 10, 4, embedding_name="a"), maxlen=5)
    assert (v.combiner, v.length_name, v.weight_name, v.weight_norm) == ("mean", None, None, True)   # :60-66
    assert (v.name, v.vocabulary_size, v.embedding_dim, v.embedding_name) == ("h", 10, 4, "a")
    d = DenseFeat("d")
    assert (d.dimension, d.dtype, d.transform_fn) == (1, "float32", None)
    assert hash(s) == hash("a")


def test_build_input_features_ordering_and_shapes():
    # deepctr/feature_column.py:145-168: the input ordering contract
    cols = [SparseFeat("s", 10, 4), DenseFeat("d", 3),
            VarLenSparseFeat(SparseFeat("v", 10, 4), maxlen=7, length_name="len", weight_name="w")]
    feats = build_input_features(cols)
    assert list(feats) == ["s", "d", "v", "w", "len"] == get_feature_names(cols)
    assert feats["s"].shape == (None, 1) and feats["d"].shape == (None, 3)
    assert feats["v"].shape == (None, 7) and feats["w"].shape == (None, 7, 1) and feats["len"].shape == (None, 1)
    assert feats["len"].dtype == "int32" and feats["w"].dtype == "float32"
    with pytest.raises(TypeError):
        build_input_features([object()])
    # duplicated columns across linear + dnn collapse by name (App. F.1)
    assert get_feature_names(cols + cols) == ["s", "d", "v", "w", "len"]


def test_string_feature_requires_hash():
    with pytest.raises(ValueError, match="requires use_hash=True"):
        build_input_features([SparseFeat("s", 10, 4, dtype="string")])
    build_input_features([SparseFeat("s", 10, 4, dtype="string", use_hash=True)])


def test_shared_embedding_table_naming_and_compat():
    # tests/feature_test.py:35-60
    cols = [SparseFeat("item_id", 11, 8),
            VarLenSparseFeat(SparseFeat("hist_item_id", 11, 8, embedding_name="item_id"), maxlen=4,
                             length_name="seq_length")]
    model = DIN(cols, ["item_id"], dnn_hidden_units=(4,), att_hidden_size=(3,))
    names = [l.name for l in model.layers]
    assert "sparse_emb_item_id" in names and "sparse_seq_emb_hist_item_id" not in names
    assert model.get_layer("sparse_emb_item_id").mask_zero
    bad = [SparseFeat("item", 10, 4), VarLenSparseFeat(SparseFeat("hist", 11, 4, embedding_name="item"), 3)]
    with pytest.raises(ValueError, match="same embedding_name"):
        DeepFM(bad, bad)


def test_dense_not_supported_flag():
    cols = _criteo()
    feats = build_input_features(cols)
    with pytest.raises(ValueError, match="DenseFeat is not supported"):
        input_from_feature_columns(feats, cols, 0, 1024, support_dense=False)


def test_deepfm_graph_weights_and_planner_layout():
    cols = _criteo(n_sparse=4, n_dense=3, dim=8)
    model = DeepFM(cols, cols, dnn_hidden_units=(16, 8))
    names = [w.name for w in model.weights]
    # reference weight naming (SURVEY.md section 5)
    for f in range(4):
        assert "linear0sparse_emb_C%d/embeddings" % f in names and "sparse_emb_C%d/embeddings" % f in names
    assert any(n.endswith("linear_kernel") for n in names) and any(n.endswith("global_bias") for n in names)
    assert any(n.endswith("kernel0") for n in names) and any(n.endswith("bias1") for n in names)
    shapes = {w.name: w.shape for w in model.weights}
    assert shapes["sparse_emb_C2/embeddings"] == (12, 8) and shapes["linear0sparse_emb_C2/embeddings"] == (12, 1)
    dnn_k0 = [w for w in model.weights if w.name.endswith("/kernel0") and len(w.shape) == 2 and w.shape[1] == 16][0]
    assert dnn_k0.shape == (4 * 8 + 3, 16)                       # [sparse embs | dense] ordering (App. F.5)
    p = model.planner
    assert len(p.slots) == 8 and p.main_width == 32 and p.lin_width == 4 and p.fast and p.fast_n == 4
    assert p.main_ld % 4 == 0 and p.main_ld >= 32 + 3             # room for the dense tail, 16 B rows
    assert [s.col for s in p.main] == [0, 8, 16, 24]
    assert model.count_params() == sum(int(np.prod(s)) for s in shapes.values())
    # initial values: embeddings N(0, 1e-4), linear tables zeros, biases zeros
    w = {x.name: x for x in model.weights}
    assert np.all(w["linear0sparse_emb_C0/embeddings"].value() == 0)
    assert 0 < np.abs(w["sparse_emb_C0/embeddings"].value()).max() < 1e-3


def test_builders_construct_and_validate_arguments():
    cols = _criteo()
    assert xDeepFM(cols, cols, cin_layer_size=(8, 4)).outputs.shape == (None, 1)
    assert xDeepFM(cols, cols, cin_layer_size=()).outputs.shape == (None, 1)
    with pytest.raises(ValueError, match="even number"):
        xDeepFM(cols, cols, cin_layer_size=(7, 4), cin_split_half=True)
    assert DCN(cols, cols, cross_num=2).outputs.shape == (None, 1)
    assert DCN([], cols, cross_num=1, dnn_hidden_units=()).outputs.shape == (None, 1)
    with pytest.raises(ValueError, match="Either hidden_layer or cross layer"):
        DCN(cols, cols, cross_num=0, dnn_hidden_units=())
    assert AutoInt(cols, cols).outputs.shape == (None, 1)
    with pytest.raises(ValueError, match="Either hidden_layer or att_layer_num"):
        AutoInt(cols, cols, att_layer_num=0, dnn_hidden_units=())
    # DCN / AutoInt take model inputs from dnn_feature_columns only (App. F.11)
    assert DCN(cols[:2], cols).input_names == get_feature_names(cols)


def test_varlen_pooling_chains_are_folded_into_the_fused_gather():
    cols = [SparseFeat("s", 20, 4),
            VarLenSparseFeat(SparseFeat("a", 12, 4), maxlen=5, combiner="sum", length_name="la"),
            VarLenSparseFeat(SparseFeat("b", 12, 4), maxlen=5, combiner="mean"),
            VarLenSparseFeat(SparseFeat("c", 12, 4, use_hash=True), maxlen=5, combiner="max", length_name="la",
                             weight_name="wc")]
    model = DeepFM(cols, cols, dnn_hidden_units=(4,))
    from deepctr_b200 import _lib as L
    by = {s.input_name + ("/lin" if s.dim == 1 else ""): s for s in model.planner.slots}
    assert by["a"].pool == L.POOL_SUM and by["a"].mask_mode == L.MASK_LENGTH and by["a"].len_name == "la"
    assert by["b"].pool == L.POOL_MEAN and by["b"].mask_mode == L.MASK_ZERO_ID
    assert by["c"].pool == L.POOL_MAX and by["c"].weight_mode == L.WEIGHT_SOFTMAX and by["c"].weight_name == "wc"
    assert by["c"].hash[0] == L.HASH_FARM_MASK_ZERO
    assert by["s"].pool == L.POOL_NONE and by["s"].maxlen == 1
    assert len(model.planner.slots) == 8 and not model.planner.seq     # no [B,T,E] tensor is ever materialised


def test_layer_configs_roundtrip():
    from deepctr_b200 import layers as LY
    for layer in [LY.CIN((8, 4), "relu", True), LY.CrossNet(2, "matrix"), LY.InteractingLayer(4, 2, False),
                  LY.DNN((4, 2), "relu"), LY.PredictionLayer("regression"), LY.SequencePoolingLayer("max", True),
                  LY.AttentionSequencePoolingLayer((4, 2), "dice", True), LY.Linear(0.1, 2, True),
                  LY.Hash(5, True), LY.Dice()]:
        cfg = layer.get_config()
        clone = layer.__class__.from_config({k: v for k, v in cfg.items() if k != "trainable"})
        assert clone.get_config().keys() == cfg.keys()
    assert set(LY.custom_objects) >= {"FM", "CIN", "CrossNet", "InteractingLayer", "DNN", "Dice", "Hash", "Linear"}
    with pytest.raises(ValueError):
        LY.InteractingLayer(head_num=0)
    with pytest.raises(ValueError):
        LY.SequencePoolingLayer("median")
    with pytest.raises(ValueError):
        LY.CIN(())


def test_compute_path_fails_loudly_without_cuda():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from deepctr_b200._lib import B2ctrError
    cols = _criteo()
    model = DeepFM(cols, cols, dnn_hidden_units=(4,))
    model.compile("sgd", "binary_crossentropy")
    x = {c.name: np.zeros(4, np.int32 if c.name[0] == "C" else np.float32) for c in cols}
    with pytest.raises(B2ctrError, match="no CPU fallback|CUDA"):
        model.predict(x, batch_size=4)


def test_host_pack_native_thread_pool():
    """b2ctr_host_pack (host-only entry point of the C-ABI): blocks land at their offsets, for the inline
    path (small), the pooled path (large, split across workers inside blocks) and empty input."""
    import ctypes as C
    from deepctr_b200 import _lib as L
    rng = np.random.RandomState(0)
    for sizes, threads in [([10, 0, 7], 0), ([300000, 1, 65536 * 4, 12345, 65536 * 8], 0),
                           ([1 << 20, 1 << 20, 3], 3), ([1 << 21], 1), ([], 0)]:
        blocks = [rng.randint(0, 255, s).astype(np.uint8) for s in sizes]
        n = len(blocks)
        gap = 5
        offs, off = [], 0
        for s in sizes:
            offs.append(off)
            off += s + gap
        dst = np.full(off + 1, 255, np.uint8)
        src = (C.c_void_p * max(n, 1))(*[b.ctypes.data for b in blocks])
        nb = (C.c_int64 * max(n, 1))(*sizes)
        of = (C.c_int64 * max(n, 1))(*offs)
        L.check(L.lib().b2ctr_host_pack(src, nb, of, n, C.c_void_p(dst.ctypes.data), threads), "host_pack")
        for b, o in zip(blocks, offs):
            assert (dst[o:o + len(b)] == b).all()
            assert (dst[o + len(b):o + len(b) + gap] == 255).all()      # nothing written between blocks
    with pytest.raises(ValueError):
        L.check(L.lib().b2ctr_host_pack(None, None, None, 2, None, 0), "host_pack")


def test_dense_gemm_policy_helpers():
    """Pure host logic of ops.dense: split-K sizing for CTA-pair tiles and the conditions under which the
    producer of dZ can write its operand planes itself."""
    from deepctr_b200 import ops, kernels as K
    assert ops._split_k(845, 256, 65536) == 18            # 4 pair tiles x 18 K slices = 72 of 74 SM pairs
    assert ops._split_k(256, 128, 65536) == 64            # one tile: capped by K / 1024
    assert ops._split_k(64, 1, 65536) == 256               # skinny wgrad: ~256-row slices, up to 592 CTAs
    assert ops._split_k(845, 1, 65536) == 42               # 14 column blocks x 42 slices = 588 CTAs
    assert ops._split_k(845, 256, 2048) == 1              # short reductions are not split
    assert ops._split_k(30000, 30000, 1 << 20) == 1       # more tiles than SM pairs
    assert K.planes_fusable(65536, 256) and K.planes_fusable(65536, 128) and K.planes_fusable(65536, 64)
    assert not K.planes_fusable(65536, 1) and not K.planes_fusable(65537, 256) and not K.planes_fusable(256, 96)
    assert not K.planes_fusable(256, 2048)                # wider than one vectorised row group
    assert ops.GEMM_PRECISION == __import__("deepctr_b200._lib", fromlist=["x"]).GEMM_BF16X3


def test_shard_transport_choice():
    """row-sharded tables: peer mappings up to ~0.4 TB of peer-mapped rows, NCCL all-to-all beyond (DESIGN.md section 9)"""
    from deepctr_b200 import parallel
    c2 = 26 * 1000000 * 33 * 4                    # C2: 3.4 GB of tables in total
    assert parallel.choose_transport(c2 // 8, 8) == "peer"
    c5 = 26 * 12500000 * 129 * 4                  # C5: 167.7 GB per rank
    assert parallel.choose_transport(c5, 2) == "peer"      # measured: full rate
    assert parallel.choose_transport(c5, 8) == "a2a"       # measured: peer 17.6 ms, all-to-all 4.2 ms per step
    assert parallel.choose_transport(c5, 1) == "peer"


@pytest.mark.parametrize("fields,heads,att", [(64, 2, 32), (65, 1, 8), (4, 1, 33), (64, 4, 13)])
def test_interacting_layer_rejects_unsupported_shapes_at_build(fields, heads, att):
    """F <= 64, att_embedding_size <= 32 and F * head_num * att_embedding_size <= 3072 (the attention backward's
    shared memory): a shape outside is refused when the layer is built, not at the first training step"""
    from deepctr_b200.layers import InteractingLayer
    with pytest.raises(ValueError, match="InteractingLayer supports"):
        InteractingLayer(att_embedding_size=att, head_num=heads).build((None, fields, 16))


def test_interacting_layer_builds_at_the_bound():
    from deepctr_b200.layers import InteractingLayer
    layer = InteractingLayer(att_embedding_size=16, head_num=3)
    layer.build((None, 64, 16))
    assert layer.built
