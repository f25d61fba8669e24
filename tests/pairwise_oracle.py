"""TEST INFRASTRUCTURE - CPU restatement (torch-CPU fp32, autograd for gradients) of the reference's NFM and AFM:
BiInteractionPooling (deepctr/layers/interaction.py:196-201), AFMLayer (:122-146) and the builder bodies
deepctr/models/nfm.py:37-61 and deepctr/models/afm.py:39-61, composed from the helpers of oracle/ops.py and
oracle/models.py (feature-column lookups, linear logit, DNN, prediction).  Pinned by the fixtures that the reference's
own code produced (tests/golden/generate_pairwise.py, checked in tests/test_pairwise_goldens.py).
"""
import torch

from oracle import models as OM
from oracle import ops as O


# ---- BiInteractionPooling (layers/interaction.py:196-201) ------------------------------------------
def bi_interaction(x):
    square_of_sum = x.sum(dim=1, keepdim=True) ** 2
    sum_of_square = (x * x).sum(dim=1, keepdim=True)
    return 0.5 * (square_of_sum - sum_of_square)             # [B,1,E]


# ---- AFMLayer (layers/interaction.py:122-146), literal op sequence ----------------------------------
def afm(embeds, attention_W, attention_b, projection_h, projection_p=None):
    """embeds: list of F [B,1,E] tensors (or one [B,F,E]).  Returns the attention output [B,E], or the layer output
    [B,1] when projection_p is given (the dropout is the identity outside training)."""
    if isinstance(embeds, torch.Tensor):
        embeds = list(torch.split(embeds, 1, dim=1))
    row, col = [], []
    for i in range(len(embeds)):                             # itertools.combinations order   :126-128
        for j in range(i + 1, len(embeds)):
            row.append(embeds[i])
            col.append(embeds[j])
    p = torch.cat(row, dim=1)                                # [B,P,E]                       :130
    q = torch.cat(col, dim=1)
    bi = p * q                                               # :132
    temp = torch.relu(torch.tensordot(bi, attention_W, dims=([-1], [0])) + attention_b)     # :135-136
    score = torch.softmax(torch.tensordot(temp, projection_h, dims=([-1], [0])), dim=1)     # :138-139
    att = (score * bi).sum(dim=1)                            # :140-141
    if projection_p is None:
        return att
    return torch.tensordot(att, projection_p, dims=([-1], [0]))                             # :145


# ---- builders ------------------------------------------------------------------------------------
def nfm(inputs, linear_cols, dnn_cols, W, task="binary", dnn_activation="relu"):
    """deepctr/models/nfm.py:37-61 (bi_dropout is the identity outside training).  W as for oracle.models.deepfm;
    an empty dnn_kernels list is the dnn_hidden_units=() case."""
    lin = OM.linear_logit(inputs, linear_cols, W["tables"], W.get("linear_kernel"))
    embs, dense = OM.input_from_feature_columns(inputs, dnn_cols, W["tables"])
    bi_out = bi_interaction(torch.cat(embs, dim=1))                                  # :48-49
    h = O.dnn(OM.combined_dnn_input([bi_out], dense), W["dnn_kernels"], W["dnn_biases"], dnn_activation)  # :52-53
    logit = lin + h @ W["dense_kernel"]                                              # :54-56
    return logit, O.prediction(logit, W.get("global_bias"), task)


def afm_model(inputs, linear_cols, dnn_cols, W, fm_group="default_group", use_attention=True, task="binary"):
    """deepctr/models/afm.py:39-61.  W['afm']: one dict (attention_W, attention_b, projection_h, projection_p) per
    group selected by ``k in fm_group``, in group order."""
    groups, _ = OM.input_from_feature_columns(inputs, dnn_cols, W["tables"], support_group=True)
    lin = OM.linear_logit(inputs, linear_cols, W["tables"], W.get("linear_kernel"))
    chosen = [v for k, v in groups.items() if k in fm_group]
    if use_attention:
        parts = [afm(v, **lw) for v, lw in zip(chosen, W["afm"])]                     # :50-52
    else:
        parts = [O.fm(torch.cat(v, dim=1)) for v in chosen]                           # :53-55
    logit = lin
    for f in parts:
        logit = logit + f
    return logit, O.prediction(logit, W.get("global_bias"), task)
