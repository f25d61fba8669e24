"""TEST INFRASTRUCTURE - CPU restatement (torch-CPU fp32, autograd for gradients) of the reference's builder bodies
deepctr/models/ifm.py:40-74 and deepctr/models/difm.py:43-82, with the refined first-order term of
deepctr/feature_column.py:171-210 (sparse_feat_refine_weight), composed from the helpers of oracle/ops.py and
oracle/models.py.  Pinned by the fixtures that the reference's own code produced (tests/golden/generate_ifm.py, checked
in tests/test_ifm_goldens.py).
"""
import torch

from oracle import models as OM
from oracle import ops as O


def refined_linear(inputs, linear_cols, W, m):
    """get_linear_logit with sparse_feat_refine_weight=m: the dim-1 lookups concatenated on the last axis [B,1,F]
    times expand_dims(m, 1), then Linear mode 0 / 2 (the dense kernel term is not reweighted)."""
    class _One(object):
        def __init__(self, fc):
            self._fc = fc

        def __getattr__(self, k):
            return 1 if k == "embedding_dim" else getattr(self._fc, k)

    cols = []
    for fc in linear_cols:
        kind = OM._kind(fc)
        if kind == "dense":
            cols.append(fc)
        else:
            w = _One(fc)
            if kind == "varlen":
                w.sparsefeat = fc.sparsefeat
            cols.append(w)
    embs, dense = OM.input_from_feature_columns(inputs, cols, W["tables"], prefix="linear0")
    sparse_in = torch.cat(embs, dim=-1) * m.unsqueeze(1) if embs else None           # :193-200
    dense_in = torch.cat(dense, dim=-1) if dense else None
    return O.linear(sparse_in, dense_in, W.get("linear_kernel"))


def _tail(inputs, linear_cols, embs, W, m, task):
    lin = refined_linear(inputs, linear_cols, W, m)                                    # ifm.py:62-63
    fm_logit = O.fm(torch.cat(embs, dim=1) * m.unsqueeze(-1))                           # :65-68
    logit = lin + fm_logit                                                              # :70
    return logit, O.prediction(logit, W.get("global_bias"), task)


def ifm(inputs, linear_cols, dnn_cols, W, task="binary", dnn_activation="relu"):
    """W as for oracle.models.deepfm (tables, linear_kernel, dnn_kernels / dnn_biases) plus W['m_kernels'] = [the
    Dense(F) kernel]."""
    embs, _ = OM.input_from_feature_columns(inputs, dnn_cols, W["tables"])              # :50-51
    h = O.dnn(OM.combined_dnn_input(embs, []), W["dnn_kernels"], W["dnn_biases"], dnn_activation)   # :55-56
    z = h @ W["m_kernels"][0]                                                           # :58
    m = z.shape[-1] * torch.softmax(z, dim=1)                                           # :60
    return _tail(inputs, linear_cols, embs, W, m, task)


def difm(inputs, linear_cols, dnn_cols, W, att_embedding_size=8, att_head_num=8, att_res=True, task="binary",
         dnn_activation="relu"):
    """W as for ifm, plus W['att'] = [InteractingLayer weights]; W['m_kernels'] = [m_vec kernel, m_bit kernel]."""
    embs, _ = OM.input_from_feature_columns(inputs, dnn_cols, W["tables"])              # :53-54
    lw = W["att"][0]
    att = O.interacting(torch.cat(embs, dim=1), lw["query"], lw["key"], lw["value"], lw.get("res"), att_head_num,
                        att_embedding_size, att_res, scaling=True)                     # :59-60
    m_vec = att.flatten(1) @ W["m_kernels"][0]                                          # :61-62
    h = O.dnn(OM.combined_dnn_input(embs, []), W["dnn_kernels"], W["dnn_biases"], dnn_activation)   # :64-65
    m_bit = h @ W["m_kernels"][1]                                                       # :66
    return _tail(inputs, linear_cols, embs, W, m_vec + m_bit, task)                    # :68
