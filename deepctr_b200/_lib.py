"""ctypes binding of ``libb2ctr.so`` (the C-ABI declared in ``include/b2ctr.h``).

This is the only place Python touches native code.  There is NO fallback: if the shared library
is missing or a symbol cannot be resolved, importing the compute path raises.  PyTorch is used
by callers purely as the owner of device memory and streams; only raw pointers cross this line.
"""
import ctypes as C
import os
import subprocess

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libb2ctr.so")
CSRC = os.path.join(_HERE, "csrc")

# ---- enums (mirror include/b2ctr.h) ---------------------------------------------------------
OK, ERR_INVALID_ARG, ERR_CUDA, ERR_UNSUPPORTED, ERR_WORKSPACE = 0, -1, -2, -3, -4
IDX_I32, IDX_I64 = 0, 1
POOL_NONE, POOL_SUM, POOL_MEAN, POOL_MAX = 0, 1, 2, 3
MASK_NONE, MASK_ZERO_ID, MASK_LENGTH = 0, 1, 2
HASH_NONE, HASH_FARM, HASH_FARM_MASK_ZERO = 0, 1, 2
WEIGHT_NONE, WEIGHT_RAW, WEIGHT_SOFTMAX = 0, 1, 2
ACT_NONE, ACT_RELU, ACT_SIGMOID, ACT_TANH = 0, 1, 2, 3
GEMM_FP32, GEMM_BF16X3 = 0, 1
TASK_BINARY, TASK_REGRESSION = 0, 1
UNIFORM_STORE_GRADS = 1

ACT_BY_NAME = {None: ACT_NONE, "linear": ACT_NONE, "relu": ACT_RELU, "sigmoid": ACT_SIGMOID,
               "tanh": ACT_TANH}
POOL_BY_NAME = {"sum": POOL_SUM, "mean": POOL_MEAN, "max": POOL_MAX}


class Feature(C.Structure):
    """b2ctr_feature_t"""
    _fields_ = [("table", C.c_void_p), ("idx", C.c_void_p), ("len", C.c_void_p),
                ("weight", C.c_void_p), ("out", C.c_void_p),
                ("vocab", C.c_int64), ("idx_stride", C.c_int64), ("out_ld", C.c_int64),
                ("out_col", C.c_int32), ("dim", C.c_int32), ("maxlen", C.c_int32),
                ("idx_dtype", C.c_int32), ("pool", C.c_int32), ("mask_mode", C.c_int32),
                ("hash_mode", C.c_int32), ("weight_mode", C.c_int32), ("src_table", C.c_void_p),
                ("len_stride", C.c_int32), ("weight_ld", C.c_int32)]


class UniformGather(C.Structure):
    """b2ctr_uniform_gather_t"""
    _fields_ = [("feats", C.POINTER(Feature)), ("lin_tables", C.POINTER(C.c_void_p)),
                ("dense", C.c_void_p), ("x", C.c_void_p), ("linear", C.c_void_p), ("fm", C.c_void_p),
                ("ldx", C.c_int64), ("dense_ld", C.c_int64), ("x_cols", C.c_int64),
                ("nfeat", C.c_int32),
                ("ndense", C.c_int32), ("fm_mask", C.c_uint64 * 2), ("flags", C.c_int32), ("world", C.c_int32),
                ("peer_tables", C.c_void_p), ("peer_lin_tables", C.c_void_p)]


class FfmField(C.Structure):
    """b2ctr_ffm_field_t"""
    _fields_ = [("idx", C.c_void_p), ("pooled", C.c_void_p), ("grad", C.c_void_p), ("idx_stride", C.c_int64),
                ("vocab", C.c_int64), ("pooled_ld", C.c_int64), ("grad_ld", C.c_int64), ("idx_dtype", C.c_int32),
                ("hash_mode", C.c_int32)]


class Gemm(C.Structure):
    """b2ctr_gemm_t"""
    _fields_ = [("a", C.c_void_p), ("b", C.c_void_p), ("c", C.c_void_p), ("bias", C.c_void_p),
                ("m", C.c_int64), ("n", C.c_int64), ("k", C.c_int64),
                ("lda", C.c_int64), ("ldb", C.c_int64), ("ldc", C.c_int64),
                ("trans_a", C.c_int32), ("trans_b", C.c_int32), ("act", C.c_int32),
                ("accumulate", C.c_int32), ("precision", C.c_int32), ("split_k", C.c_int32),
                ("alpha", C.c_float), ("variant", C.c_int32), ("a_planes", C.c_void_p), ("b_planes", C.c_void_p)]


class CinGemm(C.Structure):
    """b2ctr_cin_gemm_t"""
    _fields_ = [("t0", C.c_void_p), ("ld0", C.c_int64), ("xk", C.c_void_p), ("ldk", C.c_int64), ("rows", C.c_int64),
                ("m", C.c_int32), ("h", C.c_int32), ("hp", C.c_int32), ("n", C.c_int32),
                ("w_planes", C.c_void_p), ("dy_planes", C.c_void_p), ("c", C.c_void_p), ("ldc", C.c_int64),
                ("bias", C.c_void_p), ("act", C.c_int32), ("mode", C.c_int32), ("split_k", C.c_int32)]


class AttGemm(C.Structure):
    """b2ctr_att_gemm_t"""
    _fields_ = [("query", C.c_void_p), ("ldq", C.c_int64), ("keys", C.c_void_p), ("key_batch_stride", C.c_int64),
                ("batch", C.c_int64), ("maxlen", C.c_int32), ("dim", C.c_int32), ("n", C.c_int32),
                ("planes", C.c_void_p), ("c", C.c_void_p), ("ldc", C.c_int64), ("bias", C.c_void_p),
                ("act", C.c_int32), ("mode", C.c_int32), ("split_k", C.c_int32)]


class Mha(C.Structure):
    """b2ctr_mha_t"""
    _fields_ = [("q", C.c_void_p), ("ldq", C.c_int64), ("k", C.c_void_p), ("ldk", C.c_int64),
                ("v", C.c_void_p), ("ldv", C.c_int64), ("res", C.c_void_p), ("ldr", C.c_int64),
                ("out", C.c_void_p), ("ldo", C.c_int64), ("stats", C.c_void_p),
                ("qlen", C.c_void_p), ("klen", C.c_void_p), ("qmask", C.c_void_p), ("kmask", C.c_void_p),
                ("batch", C.c_int64), ("T", C.c_int32), ("heads", C.c_int32), ("d", C.c_int32),
                ("scale", C.c_float), ("blinding", C.c_int32), ("dropout_rate", C.c_float), ("seed", C.c_uint64),
                ("dout", C.c_void_p), ("lddo", C.c_int64), ("dq", C.c_void_p), ("lddq", C.c_int64),
                ("dk", C.c_void_p), ("lddk", C.c_int64), ("dv", C.c_void_p), ("lddv", C.c_int64)]


class Regulate(C.Structure):
    """b2ctr_regulate_t"""
    _fields_ = [("mode", C.c_int32), ("nfield", C.c_int32), ("dim", C.c_int32), ("dx_accumulate", C.c_int32),
                ("batch", C.c_int64), ("x", C.c_void_p), ("ldx", C.c_int64), ("h", C.c_void_p), ("ldh", C.c_int64),
                ("ax", C.c_void_p), ("ldax", C.c_int64), ("ah", C.c_void_p), ("ldah", C.c_int64),
                ("g0", C.c_void_p), ("g1", C.c_void_p), ("inv_tau0", C.c_float), ("inv_tau1", C.c_float),
                ("u", C.c_void_p), ("ldu", C.c_int64), ("ucol", C.c_int64),
                ("y0", C.c_void_p), ("ldy0", C.c_int64), ("y0col", C.c_int64),
                ("y1", C.c_void_p), ("ldy1", C.c_int64), ("y1col", C.c_int64),
                ("dx", C.c_void_p), ("lddx", C.c_int64), ("dh", C.c_void_p), ("lddh", C.c_int64),
                ("dax", C.c_void_p), ("lddax", C.c_int64), ("dah", C.c_void_p), ("lddah", C.c_int64),
                ("dg0", C.c_void_p), ("dg1", C.c_void_p)]



CONV_STACK_MAX_STAGES = 8          # b2ctr.h B2CTR_CONV_STACK_MAX_STAGES
CONV_STAGE_CONV, CONV_STAGE_KMAX = 0, 1


class ConvStage(C.Structure):
    """b2ctr_conv_stage_t"""
    _fields_ = [("kind", C.c_int32), ("width", C.c_int32), ("filters", C.c_int32), ("act", C.c_int32),
                ("k", C.c_int32), ("reserved", C.c_int32), ("kernel", C.c_void_p), ("bias", C.c_void_p),
                ("dkernel", C.c_void_p), ("dbias", C.c_void_p)]


class ConvStack(C.Structure):
    """b2ctr_conv_stack_t"""
    _fields_ = [("struct_size", C.c_int32), ("nstage", C.c_int32), ("rows", C.c_int32), ("dim", C.c_int32),
                ("channels", C.c_int32), ("dx_accumulate", C.c_int32), ("batch", C.c_int64),
                ("x", C.c_void_p), ("ldx", C.c_int64), ("xcol", C.c_int64),
                ("out", C.c_void_p), ("ldout", C.c_int64), ("outcol", C.c_int64),
                ("dx", C.c_void_p), ("lddx", C.c_int64), ("dxcol", C.c_int64),
                ("stage", ConvStage * CONV_STACK_MAX_STAGES)]

FWBI_MAX_FIELDS, FWBI_MAX_GROUPS = 256, 8   # b2ctr.h B2CTR_FWBI_MAX_FIELDS / _GROUPS


class FieldWiseBi(C.Structure):
    """b2ctr_field_wise_bi_t"""
    _fields_ = [("struct_size", C.c_int32), ("nfield", C.c_int32), ("ngroup", C.c_int32), ("dim", C.c_int32),
                ("dx_accumulate", C.c_int32), ("reserved", C.c_int32), ("batch", C.c_int64),
                ("x", C.c_void_p), ("ldx", C.c_int64),
                ("col", C.c_int64 * FWBI_MAX_FIELDS), ("group", C.c_int32 * FWBI_MAX_FIELDS),
                ("kernel_mf", C.c_void_p), ("kernel_fm", C.c_void_p), ("bias_mf", C.c_void_p), ("bias_fm", C.c_void_p),
                ("out", C.c_void_p), ("ldout", C.c_int64), ("outcol", C.c_int64),
                ("dx", C.c_void_p), ("lddx", C.c_int64),
                ("dkernel_mf", C.c_void_p), ("dkernel_fm", C.c_void_p), ("dbias_mf", C.c_void_p),
                ("dbias_fm", C.c_void_p)]


_vp, _i32, _i64, _f32, _sz, _u64 = C.c_void_p, C.c_int32, C.c_int64, C.c_float, C.c_size_t, C.c_uint64

# name -> (restype, argtypes).  Must list every symbol of include/b2ctr.h (tests check this).
SIGNATURES = {
    "b2ctr_abi_version": (_i32, []),
    "b2ctr_last_error": (C.c_char_p, []),
    "b2ctr_launch_count": (_i64, []),
    "b2ctr_reset_launch_count": (None, []),
    "b2ctr_embed_gather_fwd": (_i32, [C.POINTER(Feature), _i32, _i64, _vp]),
    "b2ctr_embed_scatter_add": (_i32, [C.POINTER(Feature), _i32, _i64, _f32, _vp]),
    "b2ctr_embed_max_pool_shares": (_i32, [C.POINTER(Feature), _i32, _i64, _vp, _i64, _vp]),
    "b2ctr_embed_gather_uniform_fwd": (_i32, [C.POINTER(UniformGather), _i64, _vp]),
    "b2ctr_embed_scatter_uniform_bwd": (_i32, [C.POINTER(UniformGather), _vp, _vp, _vp, _f32, _f32,
                                               _i64, _vp]),
    "b2ctr_embed_gather_uniform_fwd_ex": (_i32, [C.POINTER(UniformGather), _vp, _vp, _i64, _i64, _vp]),
    "b2ctr_embed_scatter_uniform_bwd_ex": (_i32, [C.POINTER(UniformGather), _vp, _vp, _vp, _vp, _f32, _f32,
                                                  _i64, _vp]),
    "b2ctr_embed_oob_count": (_i32, [C.POINTER(C.c_int64), _i32, _vp]),
    "b2ctr_embed_update_sorted_workspace_bytes": (_sz, [_i32, _i32, _i64]),
    "b2ctr_embed_update_sorted": (_i32, [C.POINTER(UniformGather), _vp, _vp, _vp, _i32, _f32, _f32, _f32,
                                         C.POINTER(C.c_void_p), C.POINTER(C.c_void_p), _i64, _vp, _sz, _vp]),
    "b2ctr_hash64": (_i32, [_vp, _i32, _i64, _i64, _i32, _vp, _vp]),
    "b2ctr_init_normal": (_i32, [_vp, _i64, _f32, _f32, _u64, _vp]),
    "b2ctr_gemm_workspace_bytes": (_sz, [C.POINTER(Gemm)]),
    "b2ctr_enable_peer_access": (_i32, [_i32]),
    "b2ctr_host_pack": (_i32, [C.POINTER(C.c_void_p), C.POINTER(C.c_int64), C.POINTER(C.c_int64), _i32, _vp, _i32]),
    "b2ctr_gemm": (_i32, [C.POINTER(Gemm), _vp, _sz, _vp]),
    "b2ctr_planes_bytes": (_sz, [_i64, _i64]),
    "b2ctr_split_planes": (_i32, [_vp, _i64, _i64, _i64, _vp, _vp]),
    "b2ctr_mlp_relu_supported": (_i32, [C.POINTER(_i32), _i32]),
    "b2ctr_mlp_relu_fwd": (_i32, [_vp, C.POINTER(_vp), C.POINTER(_vp), C.POINTER(_vp), _vp, C.POINTER(_i32), _i32,
                                  _i64, _vp]),
    "b2ctr_mlp_relu_bwd_workspace_bytes": (_sz, [C.POINTER(_i32), _i32]),
    "b2ctr_mlp_relu_bwd": (_i32, [_vp, _vp, _vp, C.POINTER(_vp), C.POINTER(_vp), C.POINTER(_vp), C.POINTER(_vp),
                                  C.POINTER(_i32), _i32, _i64, _vp, _sz, _vp]),
    "b2ctr_bias_act_bwd_workspace_bytes": (_sz, [_i64, _i64]),
    "b2ctr_bias_act_bwd": (_i32, [_vp, _vp, _vp, _vp, _i64, _i64, _i64, _i32, _vp, _sz, _vp]),
    "b2ctr_bias_act_bwd_planes": (_i32, [_vp, _vp, _vp, _vp, _vp, _i64, _i64, _i64, _i32, _vp, _sz, _vp]),
    "b2ctr_act_fwd": (_i32, [_vp, _vp, _i64, _i32, _vp]),
    "b2ctr_add_n": (_i32, [C.POINTER(_vp), C.POINTER(_f32), _i32, _vp, _i64, _vp]),
    "b2ctr_axpy": (_i32, [_vp, _vp, _f32, _i64, _vp]),
    "b2ctr_copy2d": (_i32, [_vp, _i64, _vp, _i64, _i64, _i64, _i32, _vp]),
    "b2ctr_rowsum": (_i32, [_vp, _i64, _vp, _i64, _i64, _vp]),
    "b2ctr_pack_rows": (_i32, [_vp, C.POINTER(_i32), _i32, _i64, _vp, _i64, _vp]),
    "b2ctr_fill": (_i32, [_vp, _f32, _i64, _vp]),
    "b2ctr_mask_nonzero_and": (_i32, [_vp, _i32, _i64, _vp, _i32, _vp]),
    "b2ctr_mask_from_len": (_i32, [_vp, _i64, _i32, _vp, _vp]),
    "b2ctr_fm_fwd": (_i32, [_vp, _i64, _i32, _i32, _vp, _i64, _vp]),
    "b2ctr_fm_bwd": (_i32, [_vp, _i64, _i32, _i32, _vp, _vp, _i64, _i32, _i64, _vp]),
    "b2ctr_fm_weighted_fwd": (_i32, [_vp, _i64, _vp, _i64, _i32, _i32, _vp, _i64, _vp]),
    "b2ctr_fm_weighted_bwd": (_i32, [_vp, _i64, _vp, _i64, _i32, _i32, _vp, _vp, _i64, _i32, _vp, _i64, _i64, _vp]),
    "b2ctr_field_scale_fwd": (_i32, [_vp, _i64, _vp, _i64, _i32, _i32, _vp, _i64, _i64, _vp]),
    "b2ctr_field_scale_bwd": (_i32, [_vp, _i64, _vp, _i64, _vp, _i64, _i32, _i32, _vp, _i64, _i32, _vp, _i64, _i64,
                                     _vp]),
    "b2ctr_softmax_rows_fwd": (_i32, [_vp, _i64, _vp, _i64, _i64, _i32, _f32, _vp]),
    "b2ctr_softmax_rows_bwd": (_i32, [_vp, _i64, _vp, _i64, _vp, _i64, _i64, _i32, _f32, _vp]),
    "b2ctr_predict_loss": (_i32, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _i64, _i32, _vp]),
    "b2ctr_sgd_step": (_i32, [_vp, _vp, _f32, _f32, _i64, _vp]),
    "b2ctr_sgd_step_multi": (_i32, [C.POINTER(C.c_void_p), C.POINTER(C.c_void_p), C.POINTER(C.c_int64), C.POINTER(C.c_float), _i32, _f32, _vp]),
    "b2ctr_adam_step": (_i32, [_vp, _vp, _vp, _vp, _f32, _f32, _f32, _f32, _f32, _i64, _i64, _vp]),
    "b2ctr_adam_step_dev": (_i32, [_vp, _vp, _vp, _vp, C.c_float, C.c_float, C.c_float, C.c_float, C.c_float, _vp,
                            _i64, _vp]),
    "b2ctr_counter_add": (_i32, [_vp, _i64, _vp]),
    "b2ctr_adagrad_step": (_i32, [_vp, _vp, _vp, _f32, _f32, _f32, _i64, _vp]),
    "b2ctr_ewise": (_i32, [_i32, _vp, _vp, _vp, _vp, _i64, _i32, _vp]),
    "b2ctr_cross_vector_fwd": (_i32, [_vp, _i64, _vp, _i64, _vp, _vp, _vp, _vp, _i64, _i32, _vp]),
    "b2ctr_cross_vector_bwd": (_i32, [_vp, _i64, _vp, _vp, _vp, _vp, _vp, _vp, _i64, _i32, _vp]),
    "b2ctr_cin_outer_fwd": (_i32, [_vp, _i64, _i64, _i64, _vp, _i64, _i64, _i64, _vp, _i64, _i32, _i32, _i32,
                                   _vp]),
    "b2ctr_cin_outer_bwd": (_i32, [_vp, _vp, _i64, _i64, _i64, _vp, _i64, _i64, _i64, _vp, _i64, _i64, _i64,
                                   _i32, _vp, _i64, _i64, _i64, _i32, _i64, _i32, _i32, _i32, _i32, _vp]),
    "b2ctr_cin_filter_planes_bytes": (_sz, [_i32, _i32, _i64]),
    "b2ctr_cin_filter_planes": (_i32, [_vp, _i32, _i32, _i32, _i64, _vp, _vp]),
    "b2ctr_cin_gemm_workspace_bytes": (_sz, [C.POINTER(CinGemm)]),
    "b2ctr_cin_gemm": (_i32, [C.POINTER(CinGemm), _vp, _sz, _vp]),
    "b2ctr_att_gemm_workspace_bytes": (_sz, [C.POINTER(AttGemm)]),
    "b2ctr_att_gemm": (_i32, [C.POINTER(AttGemm), _vp, _sz, _vp]),
    "b2ctr_cin_fold": (_i32, [C.POINTER(CinGemm), _vp, _vp, _i64, _vp]),
    "b2ctr_cin_t0_bwd": (_i32, [_vp, _i64, _vp, _i64, _i64, _i64, _i32, _i64, _i32, _i32, _vp]),
    "b2ctr_cin_t0": (_i32, [_vp, _i64, _i64, _i64, _vp, _i64, _i64, _i32, _i32, _vp]),
    "b2ctr_cin_unpad_rows": (_i32, [_vp, _vp, _i32, _i32, _i32, _i64, _vp]),
    "b2ctr_cin_sum_d": (_i32, [_vp, _i64, _i32, _i32, _i32, _vp, _i64, _i32, _i64, _vp]),
    "b2ctr_cin_expand_grad": (_i32, [_vp, _i64, _i32, _i32, _i32, _vp, _i64, _i32, _vp, _i64, _i32, _i64, _vp]),
    "b2ctr_interacting_fwd": (_i32, [_vp, _vp, _vp, _vp, _vp, _i64, _i32, _i32, _i32, _i32, _vp]),
    "b2ctr_interacting_bwd": (_i32, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i64, _i32, _i32, _i32,
                                     _i32, _vp]),
    "b2ctr_bi_interaction_fwd": (_i32, [_vp, _i64, _i32, _i32, _vp, _i64, _i64, _vp]),
    "b2ctr_bi_interaction_bwd": (_i32, [_vp, _i64, _i32, _i32, _vp, _i64, _vp, _i64, _i64, _vp]),
    "b2ctr_afm_fwd": (_i32, [_vp, _i64, _i32, _i32, _i32, _vp, _vp, _vp, _vp, _i64, _vp, _i64, _vp]),
    "b2ctr_afm_bwd_workspace_bytes": (_sz, [_i32, _i32, _i64]),
    "b2ctr_afm_bwd": (_i32, [_vp, _i64, _vp, _i64, _i32, _i32, _i32, _vp, _vp, _vp, _vp, _vp, _i64, _vp, _i64,
                             _vp, _vp, _vp, _i64, _vp, _sz, _vp]),
    "b2ctr_senet_fwd": (_i32, [_vp, _i64, _i32, _i32, _i32, _vp, _vp, _vp, _i64, _vp, _i64, _vp]),
    "b2ctr_senet_bwd_workspace_bytes": (_sz, [_i32, _i32, _i64]),
    "b2ctr_senet_bwd": (_i32, [_vp, _i64, _vp, _i64, _i32, _i32, _i32, _vp, _vp, _vp, _vp, _i64, _vp, _vp, _i64,
                               _vp, _sz, _vp]),
    "b2ctr_bilinear_fwd": (_i32, [_vp, _i64, _i32, _i32, _i32, _vp, _vp, _i64, _i64, _i64, _i64, _vp]),
    "b2ctr_bilinear_bwd_workspace_bytes": (_sz, [_i32, _i32, _i64]),
    "b2ctr_bilinear_bwd": (_i32, [_vp, _i64, _i64, _i64, _vp, _i64, _i32, _i32, _i32, _vp, _vp, _i64, _vp, _i64,
                                  _vp, _sz, _vp]),
    "b2ctr_fwfm_fwd": (_i32, [_vp, _i64, _i32, _i32, _vp, _vp, _i64, _i64, _vp]),
    "b2ctr_fwfm_bwd_workspace_bytes": (_sz, [_i32, _i64]),
    "b2ctr_fwfm_bwd": (_i32, [_vp, _i64, _vp, _i64, _i32, _i32, _vp, _vp, _i64, _vp, _i64, _vp, _sz, _vp]),
    "b2ctr_fefm_sym": (_i32, [_vp, _i32, _i32, _vp, _vp]),
    "b2ctr_fefm_fwd": (_i32, [_vp, _i64, _i32, _i32, _vp, _vp, _i64, _i64, _i64, _vp]),
    "b2ctr_fefm_bwd_workspace_bytes": (_sz, [_i32, _i32, _i64]),
    "b2ctr_fefm_bwd": (_i32, [_vp, _i64, _i64, _vp, _i64, _i32, _i32, _vp, _vp, _i64, _vp, _i64, _vp, _sz, _vp]),
    "b2ctr_pnn_inner_fwd": (_i32, [_vp, _i64, _i32, _i32, _i32, _vp, _vp, _i64, _i64, _i64, _vp]),
    "b2ctr_pnn_inner_bwd_workspace_bytes": (_sz, [_i32, _i32, _i32, _i64]),
    "b2ctr_pnn_inner_bwd": (_i32, [_vp, _i64, _i64, _vp, _i64, _i32, _i32, _i32, _vp, _vp, _i64, _vp, _i64, _vp, _sz,
                                   _vp]),
    "b2ctr_pnn_outer_fwd": (_i32, [_vp, _i64, _i32, _i32, _vp, _vp, _i64, _i64, _i64, _vp]),
    "b2ctr_pnn_outer_bwd_workspace_bytes": (_sz, [_i32, _i32, _i64]),
    "b2ctr_pnn_outer_bwd": (_i32, [_vp, _i64, _i64, _vp, _i64, _i32, _i32, _vp, _vp, _i64, _vp, _i64, _vp, _sz, _vp]),
    "b2ctr_regulate_fwd": (_i32, [C.POINTER(Regulate), _vp]),
    "b2ctr_regulate_bwd_workspace_bytes": (_sz, [_i32, _i32, _i64]),
    "b2ctr_regulate_bwd": (_i32, [C.POINTER(Regulate), _vp, _sz, _vp]),
    "b2ctr_conv_stack_fwd": (_i32, [C.POINTER(ConvStack), _vp]),
    "b2ctr_conv_stack_bwd_workspace_bytes": (_sz, [C.POINTER(ConvStack)]),
    "b2ctr_conv_stack_bwd": (_i32, [C.POINTER(ConvStack), _vp, _sz, _vp]),
    "b2ctr_field_wise_bi_fwd": (_i32, [C.POINTER(FieldWiseBi), _vp]),
    "b2ctr_field_wise_bi_bwd_workspace_bytes": (_sz, [C.POINTER(FieldWiseBi)]),
    "b2ctr_field_wise_bi_bwd": (_i32, [C.POINTER(FieldWiseBi), _vp, _sz, _vp]),
    "b2ctr_ffm_product_fwd": (_i32, [C.POINTER(FfmField), _i32, _vp, _i32, _i32, _vp, _i64, _i32, _i64, _vp]),
    "b2ctr_ffm_product_bwd": (_i32, [C.POINTER(FfmField), _i32, _vp, _i32, _i32, _vp, _i64, _i32, _i64, _vp]),
    "b2ctr_din_att_input_fwd": (_i32, [_vp, _i64, _vp, _i64, _vp, _i64, _i32, _i32, _vp]),
    "b2ctr_din_att_input_bwd": (_i32, [_vp, _i64, _vp, _i64, _vp, _vp, _vp, _i64, _i32, _i32, _vp]),
    "b2ctr_din_pool_fwd": (_i32, [_vp, _vp, _i64, _vp, _vp, _vp, _i64, _i32, _i32, _i32, _i32, _vp]),
    "b2ctr_din_pool_bwd": (_i32, [_vp, _vp, _i64, _vp, _vp, _vp, _vp, _i64, _i32, _i32, _i32, _i32, _vp]),
    "b2ctr_seqpool_fwd": (_i32, [_vp, _vp, _vp, _vp, _i64, _i32, _i32, _i32, _vp]),
    "b2ctr_seqpool_bwd": (_i32, [_vp, _vp, _vp, _vp, _vp, _i64, _i32, _i32, _i32, _vp]),
    "b2ctr_seqweight": (_i32, [_vp, _vp, _vp, _vp, _i64, _i32, _i32, _vp]),
    "b2ctr_seqscale": (_i32, [_vp, _vp, _vp, _i64, _i32, _vp]),
    "b2ctr_colstats_workspace_bytes": (_sz, [_i64, _i64]),
    "b2ctr_colstats": (_i32, [_vp, _i64, _i64, _i64, _vp, _vp, _sz, _vp]),
    "b2ctr_moving_update": (_i32, [_vp, _vp, _f32, _i64, _vp]),
    "b2ctr_bn_apply": (_i32, [_vp, _vp, _vp, _vp, _vp, _vp, _i64, _i64, _f32, _vp]),
    "b2ctr_bn_bwd": (_i32, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i64, _i64, _f32, _i32, _vp, _sz, _vp]),
    "b2ctr_dice_fwd": (_i32, [_vp, _vp, _vp, _vp, _vp, _i64, _i64, _f32, _vp]),
    "b2ctr_dice_bwd_workspace_bytes": (_sz, [_i64, _i64]),
    "b2ctr_dice_bwd": (_i32, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _i64, _i64, _f32, _i32, _vp, _sz, _vp]),
    "b2ctr_dropout": (_i32, [_vp, _vp, _i64, _f32, _u64, _vp]),
    "b2ctr_mha_fwd": (_i32, [C.POINTER(Mha), _vp]),
    "b2ctr_mha_bwd": (_i32, [C.POINTER(Mha), _vp]),
    "b2ctr_layernorm_fwd": (_i32, [_vp, _i64, _vp, _i64, _vp, _vp, _vp, _i64, _vp, _i64, _i32, _f32, _vp]),
    "b2ctr_layernorm_bwd_workspace_bytes": (_sz, [_i64, _i32]),
    "b2ctr_layernorm_bwd": (_i32, [_vp, _i64, _vp, _i64, _vp, _vp, _vp, _i64, _vp, _i64, _vp, _vp, _i64, _i32, _vp,
                                   _sz, _vp]),
    "b2ctr_shard_bucketize": (_i32, [C.POINTER(Feature), _i32, _i64, _i32, _vp, _vp, _vp]),
    "b2ctr_shard_fill": (_i32, [C.POINTER(Feature), _i32, _i64, _i32, _vp, _vp, _vp, _vp, _vp]),
    "b2ctr_shard_gather_rows": (_i32, [C.POINTER(_vp), C.POINTER(_vp), _i32, _i32, _vp, _i64, _vp, _vp, _vp]),
    "b2ctr_shard_scatter_rows": (_i32, [C.POINTER(_vp), C.POINTER(_vp), _i32, _i32, _vp, _i64, _vp, _vp, _f32,
                                        _f32, _vp]),
}


class B2ctrError(RuntimeError):
    pass


_lib = None


def build(verbose=False):
    """Compile every CUDA source for sm_90a into deepctr_b200/libb2ctr.so (nvcc cross-compiles
    without a GPU).  Called by __graft_entry__.build()."""
    r = subprocess.run(["make", "-C", CSRC, "-j8"], capture_output=True, text=True)
    if verbose or r.returncode != 0:
        print(r.stdout[-4000:])
        print(r.stderr[-4000:])
    if r.returncode != 0:
        raise B2ctrError("building libb2ctr.so failed (see output above)")
    return LIB_PATH


def lib():
    """Load the shared library once; raise (never fall back) when it is absent."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise B2ctrError(
            "libb2ctr.so not found at %s - build it with `python __graft_entry__.py build` "
            "(there is no CPU / PyTorch fallback for the compute path)" % LIB_PATH)
    handle = C.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(handle, name)  # AttributeError if the symbol is missing: loud by design
        fn.restype = res
        fn.argtypes = args
    _lib = handle
    return _lib


def check(status, what=""):
    """Map a b2ctr_status_t to the exception class the reference would raise at that point
    (ValueError for shape/argument errors, RuntimeError otherwise; SURVEY.md §8b)."""
    if status == OK:
        return
    msg = lib().b2ctr_last_error().decode("utf-8", "replace")
    if status == ERR_INVALID_ARG:
        raise ValueError("%s: %s" % (what or "b2ctr", msg))
    raise B2ctrError("%s failed (status %d): %s" % (what or "b2ctr", status, msg))


def launch_count():
    return int(lib().b2ctr_launch_count())


def reset_launch_count():
    lib().b2ctr_reset_launch_count()
