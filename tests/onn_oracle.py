"""TEST INFRASTRUCTURE - CPU restatement (torch-CPU fp32, autograd for gradients) of the reference's builder body
deepctr/models/onn.py:52-110 (ONN / NFFM), composed from the helpers of oracle/ops.py and oracle/models.py.  Pinned
by the fixtures that the reference's own code produced (tests/golden/generate_onn.py, checked in
tests/test_onn_goldens.py).
"""
import itertools

import torch

from oracle import models as OM
from oracle import ops as O


def field_lookup(inputs, fc, partner, tables):
    """feature_embedding (onn.py:113-118): field fc's row from its table for ``partner``: NoMask(Embedding(ids)) for
    a SparseFeat, SequencePoolingLayer(combiner) over the mask_zero lookup for a VarLenSparseFeat.  Hashed ids go
    through Hash(vocabulary_size) with mask_zero=False, so the sequence mask is (hashed id != 0)."""
    table = tables["sparse_emb_%s_%s" % (fc.embedding_name, partner.name)]
    ids = OM._ids(fc, inputs[fc.name], False)
    seq = O.embedding_lookup(table, ids)                                               # [B, T, E]
    if OM._kind(fc) == "sparse":
        return seq
    return O.sequence_pooling(seq, fc.combiner, mask=ids.reshape(seq.shape[:2]) != 0)


def ffm_products(inputs, dnn_cols, tables, reduce_sum=False):
    """[B, P*E] (or [B, P]): the pairwise products of onn.py:82-99, in itertools.combinations order."""
    fields = [c for c in dnn_cols if OM._kind(c) == "sparse"] + [c for c in dnn_cols if OM._kind(c) == "varlen"]
    prods = []
    for fi, fj in itertools.combinations(fields, 2):
        p = field_lookup(inputs, fi, fj, tables) * field_lookup(inputs, fj, fi, tables)   # multiply, [B, 1, E]
        prods.append(p.sum(dim=-1) if reduce_sum else p)                                  # K.sum(., axis=-1)
    return torch.cat(prods, dim=1).flatten(1)


def onn(inputs, linear_cols, dnn_cols, W, use_bn=True, reduce_sum=False, task="binary"):
    """W as for oracle.models.deepfm (tables, linear_kernel, dnn_kernels / dnn_biases, dense_kernel, global_bias)
    plus W['bn'] = {gamma, beta} of the BatchNormalization, applied in training mode (batch statistics)."""
    lin = OM.linear_logit(inputs, linear_cols, W["tables"], W.get("linear_kernel"))       # onn.py:56-57
    x = ffm_products(inputs, dnn_cols, W["tables"], reduce_sum)
    if use_bn:
        x = O.batchnorm(x, W["bn"]["gamma"], W["bn"]["beta"], training=True)              # :101-102
    _, dense = OM.input_from_feature_columns(inputs, [c for c in dnn_cols if OM._kind(c) == "dense"], {})
    h = OM.combined_dnn_input([x], dense)                                                  # :103
    if W.get("dnn_kernels"):
        h = O.dnn(h, W["dnn_kernels"], W["dnn_biases"], "relu")                           # :104
    logit = h @ W["dense_kernel"] + lin                                                     # :105-107
    return logit, O.prediction(logit, W.get("global_bias"), task)
