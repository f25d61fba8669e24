"""TEST INFRASTRUCTURE - CPU restatement (torch-CPU fp32, autograd for gradients) of the reference's FwFMLayer
(deepctr/layers/interaction.py:1393-1411), FEFMLayer (:1470-1491) and the builder bodies deepctr/models/fwfm.py:44-76
and deepctr/models/deepfefm.py:54-106, composed from the helpers of oracle/ops.py and oracle/models.py (feature-column
lookups, linear logit, DNN, prediction).  Pinned by the fixtures that the reference's own code produced
(tests/golden/generate_fefm.py, checked in tests/test_fefm_goldens.py).
"""
import itertools
from itertools import chain

import torch

from oracle import models as OM
from oracle import ops as O


# ---- FwFMLayer (layers/interaction.py:1400-1411) ---------------------------------------------------
def fwfm(x, r):
    """x [B,F,E], r [F,F] -> [B,1]; only r's upper triangle is read."""
    terms = [r[i, j] * (x[:, i] * x[:, j]).sum(dim=1, keepdim=True)                    # :1402-1408
             for i, j in itertools.combinations(range(x.shape[1]), 2)]
    return sum(terms[1:], terms[0])                                                     # :1410


# ---- FEFMLayer (layers/interaction.py:1477-1491) ---------------------------------------------------
def fefm(x, weights):
    """x [B,F,E], ``weights``: the P [E,E] field-pair matrices in itertools.combinations order -> [B,P]."""
    out = []
    for (i, j), w in zip(itertools.combinations(range(x.shape[1]), 2), weights):
        t = x[:, i] @ (w + w.t())                                                       # :1485
        out.append((t * x[:, j]).sum(dim=1, keepdim=True))                              # :1487
    return torch.cat(out, dim=1)                                                        # :1490


def _head(inputs, linear_cols, dnn_cols, W, use_linear=True):
    """(linear logit or None when it is off the output path, groups, dense values)."""
    lin = OM.linear_logit(inputs, linear_cols, W["tables"], W.get("linear_kernel")) if use_linear else None
    groups, dense = OM.input_from_feature_columns(inputs, dnn_cols, W["tables"], support_group=True)
    return lin, groups, dense


# ---- FwFM (models/fwfm.py:44-76) -------------------------------------------------------------------
def fwfm_model(inputs, linear_cols, dnn_cols, W, fm_group=("default_group",), task="binary", dnn_activation="relu"):
    """W as for oracle.models.deepfm plus W['fwfm'] = the strengths of each group selected by ``k in fm_group``, in
    group order; no dnn_kernels is the dnn_hidden_units=() case (no DNN branch)."""
    lin, groups, dense = _head(inputs, linear_cols, dnn_cols, W)                        # :46-54
    chosen = [v for k, v in groups.items() if k in fm_group]
    logit = lin
    for v, r in zip(chosen, W["fwfm"]):                                                 # :56-57
        logit = logit + fwfm(torch.cat(v, dim=1), r)
    if W.get("dnn_kernels"):                                                            # :61-67
        x = OM.combined_dnn_input(list(chain.from_iterable(groups.values())), dense)
        h = O.dnn(x, W["dnn_kernels"], W["dnn_biases"], dnn_activation)
        logit = logit + h @ W["dense_kernel"]
    return logit, O.prediction(logit, W.get("global_bias"), task)


# ---- DeepFEFM (models/deepfefm.py:54-106) ------------------------------------------------------------
def deepfefm(inputs, linear_cols, dnn_cols, W, use_fefm=True, use_linear=True, use_fefm_embed_in_dnn=True,
             exclude_feature_embed_in_dnn=False, task="binary", dnn_activation="relu"):
    """W as for oracle.models.deepfm plus W['fefm'] = the P field-pair matrices of the default group; no
    dnn_kernels is the dnn_hidden_units=() case (the DNN branch is off the output path)."""
    lin, groups, dense = _head(inputs, linear_cols, dnn_cols, W, use_linear)            # :56-62
    fefm_out = fefm(torch.cat(groups["default_group"], dim=1), W["fefm"])               # :64-67
    dnn_input = OM.combined_dnn_input(list(chain.from_iterable(groups.values())), dense)  # :69
    if use_fefm_embed_in_dnn:                                                           # :72-78
        dnn_input = fefm_out if exclude_feature_embed_in_dnn else torch.cat([dnn_input, fefm_out], dim=1)
    deep = bool(W.get("dnn_kernels"))
    parts = []
    if use_linear:
        parts.append(lin)
    if use_fefm:
        parts.append(fefm_out.sum(dim=1, keepdim=True))                                 # :84
    if deep:
        h = O.dnn(dnn_input, W["dnn_kernels"], W["dnn_biases"], dnn_activation)        # :80-82
        parts.append(h @ W["dense_kernel"])
    if not parts:
        raise NotImplementedError                                                       # :101-102
    logit = parts[0]
    for p in parts[1:]:
        logit = logit + p
    return logit, O.prediction(logit, W.get("global_bias"), task)
