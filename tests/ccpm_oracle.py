"""TEST INFRASTRUCTURE - CPU restatement (torch-CPU fp32, autograd for gradients) of the reference's builder body
deepctr/models/ccpm.py:51-81 with Keras' Conv2D ((width, 1) kernels, 'same' padding) and KMaxPooling
(deepctr/layers/sequence.py:851-864), composed from the helpers of oracle/ops.py and oracle/models.py.  Pinned by
the fixtures that the reference's own code produced (tests/golden/generate_ccpm.py, checked in
tests/test_ccpm_goldens.py).
"""
import torch

from oracle import models as OM
from oracle import ops as O

_ACT = {None: lambda v: v, "linear": lambda v: v, "relu": torch.relu, "sigmoid": torch.sigmoid, "tanh": torch.tanh}


def conv2d(x, kernel, bias, activation):
    """[B, rows, E, C] -> [B, rows, E, filters]: kernel [w, 1, C, filters], TF 'same' padding along the rows
    ((w - 1) // 2 before, the rest after), a cross-correlation."""
    w = kernel.shape[0]
    pb = (w - 1) // 2
    xp = torch.nn.functional.pad(x.permute(0, 3, 1, 2), (0, 0, pb, w - 1 - pb))
    y = torch.nn.functional.conv2d(xp, kernel.permute(3, 2, 0, 1)).permute(0, 2, 3, 1)
    if bias is not None:
        y = y + bias
    return _ACT[activation](y)


def kmax(x, k, axis):
    """The k largest values along ``axis`` in descending order, equal values lower index first."""
    vals, _ = torch.sort(x.movedim(axis, -1), dim=-1, descending=True, stable=True)
    return vals[..., :k].movedim(-1, axis)


def ccpm_k(i, l, n):
    return max(1, int((1 - pow(i / l, l - i)) * n)) if i < l else 3


def ccpm(inputs, linear_cols, dnn_cols, W, conv_kernel_width=(6, 5), conv_filters=(4, 4), task="binary"):
    """W as for oracle.models (tables, linear_kernel, dnn_kernels / dnn_biases, dense_kernel, global_bias) plus
    W['conv'], the Conv2D (kernel, bias) pairs in creation order."""
    lin = OM.linear_logit(inputs, linear_cols, W["tables"], W.get("linear_kernel"))       # ccpm.py:47-48
    embs, _ = OM.input_from_feature_columns(inputs, dnn_cols, W["tables"])               # :50-51
    n, l = len(embs), len(conv_filters)
    h = torch.cat(embs, dim=1).unsqueeze(3)                                               # :56-58
    for i in range(1, l + 1):                                                             # :60-68
        kernel, bias = W["conv"][i - 1]
        h = conv2d(h, kernel, bias, "tanh")
        h = kmax(h, min(ccpm_k(i, l, n), h.shape[1]), 1)
    x = h.flatten(1)                                                                      # :70
    x = O.dnn(x, W.get("dnn_kernels", []), W.get("dnn_biases", []), "relu")
    logit = x @ W["dense_kernel"] + lin                                                   # :71-74
    return logit, O.prediction(logit, W.get("global_bias"), task)
