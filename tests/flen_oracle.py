"""TEST INFRASTRUCTURE - CPU restatement (torch-CPU, autograd for gradients) of the reference's builder body
deepctr/models/flen.py:50-82 with its FieldWiseBiInteraction (deepctr/layers/interaction.py:1283-1337), composed
from the helpers of oracle/ops.py and oracle/models.py.  Pinned by the fixtures that the reference's own code
produced (tests/golden/generate_flen.py, checked in tests/test_flen_goldens.py).  The GPU tests run it in float64.
"""
import itertools
from itertools import chain

import torch

from oracle import models as OM
from oracle import ops as O


def field_wise_bi(groups, kernel_mf, kernel_fm, bias_mf=None, bias_fm=None):
    """G [B, F_g, E] groups -> [B, E]: sum_{g<h} kernel_mf[p] S_g S_h + bias_mf + sum_g kernel_fm[g] (S_g^2 - Q_g)
    + bias_fm, pairs in itertools.combinations order, no 1/2 on the FM term."""
    S = [g.sum(dim=1) for g in groups]
    Q = [(g * g).sum(dim=1) for g in groups]
    h_mf = sum(kernel_mf[p, 0] * S[i] * S[j]
               for p, (i, j) in enumerate(itertools.combinations(range(len(groups)), 2)))
    h_fm = sum(kernel_fm[g, 0] * (S[g] * S[g] - Q[g]) for g in range(len(groups)))
    if bias_mf is not None:
        h_mf = h_mf + bias_mf
        h_fm = h_fm + bias_fm
    return h_mf + h_fm


def flen(inputs, linear_cols, dnn_cols, W, task="binary"):
    """W as for oracle.models (tables, linear_kernel, dnn_kernels / dnn_biases, dense_kernel, global_bias) plus
    W['fwbi'] (kernel_mf, kernel_fm, bias_mf, bias_fm) and W['dnn_bn'] (the DNN's BatchNormalization gamma / beta
    per layer, or None)."""
    lin = OM.linear_logit(inputs, linear_cols, W["tables"], W.get("linear_kernel"), prefix="linear0")   # flen.py:60
    groups, dense = OM.input_from_feature_columns(inputs, dnn_cols, W["tables"], support_group=True)   # :53-58
    h = field_wise_bi([torch.cat(v, dim=1) for v in groups.values()], *W["fwbi"])                     # :66-67
    x = OM.combined_dnn_input(list(chain.from_iterable(groups.values())), dense)                      # :69-71
    x = O.dnn(x, W.get("dnn_kernels", []), W.get("dnn_biases", []), "relu", training=W["dnn_bn"] is not None,
              bn_params=W["dnn_bn"])                                                                  # :72
    logit = torch.cat([h, x], dim=-1) @ W["dense_kernel"] + lin                                       # :74-76
    return logit, O.prediction(logit, W.get("global_bias"), task)
