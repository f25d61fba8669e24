"""TEST INFRASTRUCTURE - CPU restatement (torch-CPU fp32, autograd for gradients) of the reference's
InnerProductLayer (deepctr/layers/interaction.py:655-678), OutterProductLayer (:861-921) and the builder body
deepctr/models/pnn.py:38-71, composed from the helpers of oracle/ops.py and oracle/models.py (feature-column lookups,
DNN, prediction).  Pinned by the fixtures that the reference's own code produced (tests/golden/generate_pnn.py,
checked in tests/test_pnn_goldens.py).
"""
import itertools

import torch

from oracle import models as OM
from oracle import ops as O


def _pq(x):
    """x [B,F,E] -> (p, q) [B,P,E]: the first and second field of each pair, combinations order (:665-672)."""
    rows, cols = zip(*itertools.combinations(range(x.shape[1]), 2))
    return x[:, list(rows)], x[:, list(cols)]


def inner(x, reduce_sum=True):
    """InnerProductLayer: [B,P,1] inner products, or [B,P,E] elementwise products (:674-678)."""
    p, q = _pq(x)
    out = p * q
    return out.sum(dim=2, keepdim=True) if reduce_sum else out


def outer(x, kernel, kernel_type):
    """OutterProductLayer -> [B,P].  'mat': sum_{k,l} q[k] K[k,p,l] p[l] (:881-911); 'vec' / 'num':
    sum_e p q K[p] (:915-919)."""
    p, q = _pq(x)
    if kernel_type == "mat":
        return torch.einsum("bpl,kpl,bpk->bp", p, kernel, q)
    return (p * q * kernel.unsqueeze(0)).sum(dim=-1)


def pnn(inputs, dnn_cols, W, use_inner=True, use_outter=False, kernel_type="mat", task="binary",
        dnn_activation="relu"):
    """W as for oracle.models.deepfm (tables, dnn_kernels / dnn_biases, dense_kernel) plus W['outer'] = the
    OutterProductLayer kernel when use_outter."""
    emb, dense = OM.input_from_feature_columns(inputs, dnn_cols, W["tables"])          # :44-45
    x = torch.cat(emb, dim=1)
    linear_signal = x.flatten(1)                                                        # :51-52
    parts = [linear_signal]
    if use_inner:
        parts.append(inner(x).flatten(1))                                               # :46-47
    if use_outter:
        parts.append(outer(x, W["outer"], kernel_type))                                 # :48
    deep_input = torch.cat(parts, dim=1)                                                # :54-61
    dnn_input = OM.combined_dnn_input([deep_input], dense)                              # :63
    h = O.dnn(dnn_input, W["dnn_kernels"], W["dnn_biases"], dnn_activation)            # :64
    logit = h @ W["dense_kernel"]                                                       # :65
    return logit, O.prediction(logit, W.get("global_bias"), task)                       # :67
