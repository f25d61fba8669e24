"""TEST INFRASTRUCTURE - CPU restatement (torch-CPU fp32, autograd for gradients) of the reference's FiBiNET:
SENETLayer (deepctr/layers/interaction.py:1113-1126), BilinearInteraction (:1190-1209) and the builder body
deepctr/models/fibinet.py:40-66, composed from the helpers of oracle/ops.py and oracle/models.py (feature-column
lookups, linear logit, DNN, prediction).  Pinned by the fixtures that the reference's own code produced
(tests/golden/generate_fibinet.py, checked in tests/test_fibinet_goldens.py).
"""
import itertools

import torch

from oracle import models as OM
from oracle import ops as O


# ---- SENETLayer (layers/interaction.py:1119-1126) --------------------------------------------------
def senet(x, W_1, W_2):
    """x [B,F,E] -> V [B,F,E] (the reference returns its F [B,1,E] slices)."""
    Z = x.mean(dim=-1)                                                    # :1120
    A_1 = torch.relu(torch.tensordot(Z, W_1, dims=([-1], [0])))          # :1122
    A_2 = torch.relu(torch.tensordot(A_1, W_2, dims=([-1], [0])))        # :1123
    return x * A_2.unsqueeze(2)                                           # :1124


# ---- BilinearInteraction (layers/interaction.py:1196-1209) -----------------------------------------
def bilinear(x, bilinear_type, weights):
    """x [B,F,E] -> [B,P,E]; ``weights``: [W] ('all'), F-1 ('each') or P ('interaction') [E,E] tensors."""
    v = list(torch.split(x, 1, dim=1))
    n = len(v)
    pairs = list(itertools.combinations(range(n), 2))
    if bilinear_type == "all":                                            # :1197-1199
        vid = [torch.tensordot(v[i], weights[0], dims=([-1], [0])) for i in range(n)]
        p = [vid[i] * v[j] for i, j in pairs]
    elif bilinear_type == "each":                                         # :1200-1202
        vid = [torch.tensordot(v[i], weights[i], dims=([-1], [0])) for i in range(n - 1)]
        p = [vid[i] * v[j] for i, j in pairs]
    else:                                                                 # :1203-1205
        p = [torch.tensordot(v[i], w, dims=([-1], [0])) * v[j] for (i, j), w in zip(pairs, weights)]
    return torch.cat(p, dim=1)                                            # :1208


# ---- builder (models/fibinet.py:40-66) -------------------------------------------------------------
def fibinet(inputs, linear_cols, dnn_cols, W, bilinear_type="interaction", task="binary", dnn_activation="relu"):
    """W as for oracle.models.deepfm plus W['senet'] = (W_1, W_2) and W['bilinear'] = [weights of the SENET branch's
    layer, weights of the plain branch's layer]; an empty dnn_kernels list is the dnn_hidden_units=() case."""
    lin = OM.linear_logit(inputs, linear_cols, W["tables"], W.get("linear_kernel"))        # :44-45
    embs, dense = OM.input_from_feature_columns(inputs, dnn_cols, W["tables"])            # :47-48
    x = torch.cat(embs, dim=1)
    senet_bilinear_out = bilinear(senet(x, *W["senet"]), bilinear_type, W["bilinear"][0])  # :50-54
    bilinear_out = bilinear(x, bilinear_type, W["bilinear"][1])                            # :55-56
    flat = torch.cat([senet_bilinear_out, bilinear_out], dim=-1).flatten(1)               # :58
    h = O.dnn(OM.combined_dnn_input([flat], dense), W["dnn_kernels"], W["dnn_biases"], dnn_activation)  # :59
    logit = lin + h @ W["dense_kernel"]                                                    # :60-62
    return logit, O.prediction(logit, W.get("global_bias"), task)
