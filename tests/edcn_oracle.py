"""TEST INFRASTRUCTURE - CPU restatement (torch-CPU fp32, autograd for gradients) of the reference's builder body
deepctr/models/edcn.py:55-100 with its RegulationModule (deepctr/layers/core.py:307-315) and BridgeModule
(deepctr/layers/interaction.py:1556-1565), composed from the helpers of oracle/ops.py and oracle/models.py.  Pinned by
the fixtures that the reference's own code produced (tests/golden/generate_edcn.py, checked in
tests/test_edcn_goldens.py).
"""
import torch

from oracle import models as OM
from oracle import ops as O


def regulation(x, g, inv_tau):
    """[B, F, E] * softmax_f(g * inv_tau) -> [B, F*E]."""
    return (x * torch.softmax(g * inv_tau, dim=1)).reshape(x.shape[0], -1)


def bridge(x, h, bridge_type, W):
    if bridge_type == "pointwise_addition":
        return x + h
    if bridge_type == "hadamard_product":
        return x * h
    if bridge_type == "concatenation":
        return torch.relu(torch.cat([x, h], dim=-1) @ W["dense"][0] + W["dense"][1])
    a_x = _softmax_dnn(x, *W["dense_x"])
    a_h = _softmax_dnn(h, *W["dense_h"])
    return a_x * x + a_h * h


def _softmax_dnn(x, kernels, biases):
    """DNN([d, d], 'relu', output_activation='softmax'): relu layers, then softmax over the last axis."""
    x = O.dnn(x, kernels[:-1], biases[:-1], "relu")
    return torch.softmax(x @ kernels[-1] + biases[-1], dim=-1)


def edcn(inputs, linear_cols, dnn_cols, W, cross_num=2, parameterization="vector", bridge_type="concatenation",
         tau=1.0, task="binary"):
    """W as for oracle.models.dcn (tables, dense_kernel, global_bias) plus, in creation order, W['regulation'] (the
    gates' [1, F, 1] weights), W['cross'] / W['deep'] (per layer: ([kernel], [bias]) and, for the DNN, the
    BatchNormalization's gamma / beta or None) and W['bridges'] (per layer: the nested Dense / DNN weights)."""
    lin = OM.linear_logit(inputs, linear_cols, W["tables"], W.get("linear_kernel"))        # edcn.py:60
    embs, _ = OM.input_from_feature_columns(inputs, dnn_cols, W["tables"])                # :62-63
    emb = torch.cat(embs, dim=1)                                                          # :65
    F, E = emb.shape[1], emb.shape[2]
    regs = iter(W["regulation"])
    deep_in = regulation(emb, next(regs), 1.0 / tau)                                      # :66-67
    cross_in = regulation(emb, next(regs), 1.0 / tau)
    for i in range(cross_num):
        ck, cb = W["cross"][i]
        cross_out = O.crossnet(cross_in, ck, cb, parameterization)                        # :74
        dk, db, bn = W["deep"][i]
        deep_out = O.dnn(deep_in, dk, db, "relu", training=True,
                         bn_params=[bn] if bn is not None else None)                      # :76-77
        bridge_out = bridge(cross_out, deep_out, bridge_type, W["bridges"][i])            # :79
        if i + 1 < cross_num:
            b3 = bridge_out.reshape(-1, F, E)                                              # :81
            deep_in = regulation(b3, next(regs), 1.0 / tau)
            cross_in = regulation(b3, next(regs), 1.0 / tau)
    stack = torch.cat([cross_out, deep_out, bridge_out], dim=-1)                           # :85
    logit = stack @ W["dense_kernel"] + lin                                                # :86-88
    return logit, O.prediction(logit, W.get("global_bias"), task)
