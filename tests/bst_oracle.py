"""TEST INFRASTRUCTURE - CPU restatement (torch-CPU fp32, autograd for gradients) of the reference's BST:
LayerNormalization (deepctr/layers/normalization.py:34-43), PositionEncoding (deepctr/layers/sequence.py:683-689),
Transformer (:523-635, dropout 0) and the builder body deepctr/models/sequence/bst.py:42-103, composed from the
helpers of oracle/ops.py (embedding lookup, sequence mask, attention pooling, DNN, prediction).  Pinned by the
fixtures that the reference's own code produced (tests/golden/generate_bst.py, checked in tests/test_bst_goldens.py).
"""
import torch

from oracle import ops as O

PAD = -2.0 ** 32 + 1


def layer_norm(x, gamma, beta, eps=1e-9, center=True, scale=True):
    mean = x.mean(-1, keepdim=True)                                        # :35
    var = ((x - mean) ** 2).mean(-1, keepdim=True)                         # :36
    out = (x - mean) / torch.sqrt(var + eps)                               # :37-38
    if scale:
        out = out * gamma                                                  # :39-40
    if center:
        out = out + beta                                                   # :41-42
    return out


def position_encoding(x, table, scale=True):
    out = table[None]                                                      # :685-686
    if scale:
        out = out * x.shape[-1] ** 0.5                                     # :687-688
    return out + x                                                         # :689


def transformer(queries, keys, qvalid, kvalid, W, head_num, use_positional_encoding=True, use_res=True,
                use_feed_forward=True, use_layer_norm=False, blinding=True, output_type="mean", **_):
    """W: 'query', 'key', 'value', 'fw1', 'fw2', 'ln/gamma', 'ln/beta', 'query_pe/lookup_table',
    'key_pe/lookup_table'; qvalid / kvalid bool [B, T]."""
    if use_positional_encoding:
        queries = position_encoding(queries, W["query_pe/lookup_table"])   # :540-542
        keys = position_encoding(keys, W["key_pe/lookup_table"])
    Q = torch.tensordot(queries, W["query"], dims=([-1], [0]))             # :544-547
    K = torch.tensordot(keys, W["key"], dims=([-1], [0]))
    V = torch.tensordot(keys, W["value"], dims=([-1], [0]))
    Q_, K_, V_ = (torch.cat(torch.chunk(t, head_num, dim=2), 0) for t in (Q, K, V))   # :550-552
    s = torch.matmul(Q_, K_.transpose(1, 2)) / (K_.shape[-1] ** 0.5)      # :556-558
    T = queries.shape[1]
    km = kvalid.repeat(head_num, 1)[:, None, :].expand(-1, T, -1)         # :581-585
    s = torch.where(km, s, torch.full_like(s, PAD))                        # :587-591
    if blinding:                                                           # :592-598
        eye = torch.eye(T, dtype=torch.bool)[None]
        s = torch.where(eye, torch.full_like(s, PAD), s)
    s = s - s.amax(-1, keepdim=True)                                       # :600
    p = torch.softmax(s, -1)                                               # :601
    p = p * qvalid.repeat(head_num, 1)[:, :, None].to(p.dtype)             # :602-607
    result = torch.cat(torch.chunk(torch.matmul(p, V_), head_num, dim=0), 2)   # :612-613
    if use_res:
        result = result + queries                                          # :615-617
    ln = (lambda x: layer_norm(x, W["ln/gamma"], W["ln/beta"]))
    if use_layer_norm:
        result = ln(result)                                                # :618-619
    if use_feed_forward:
        fw1 = torch.relu(torch.tensordot(result, W["fw1"], dims=([-1], [0])))   # :622
        fw2 = torch.tensordot(fw1, W["fw2"], dims=([-1], [0]))            # :624
        if use_res:
            result = result + fw2                                          # :625-626
        if use_layer_norm:
            result = ln(result)                                            # :627-628
    if output_type == "mean":
        return result.mean(1, keepdim=True)                                # :630-631
    if output_type == "sum":
        return result.sum(1, keepdim=True)                                 # :632-633
    return result


def bst(inputs, dnn_cols, history_feature_list, W, transformer_num=1, att_head_num=8, task="binary"):
    """W: 'tables' {embedding name: table}, 'transformers' [per-layer dicts as for transformer()], 'lau' (the
    attention unit's weights as for oracle.ops.attention_sequence_pooling), 'dnn_kernels', 'dnn_biases',
    'dense_kernel', 'global_bias'.  Every column is a SparseFeat, DenseFeat or a history VarLenSparseFeat."""
    def emb(fc, ids):
        return O.embedding_lookup(W["tables"][fc.embedding_name], torch.as_tensor(ids).long())

    sparse = [c for c in dnn_cols if type(c).__name__ == "SparseFeat"]
    dense = [c for c in dnn_cols if type(c).__name__ == "DenseFeat"]
    hist = [c for c in dnn_cols if type(c).__name__ == "VarLenSparseFeat"
            and c.name in ["hist_" + h for h in history_feature_list]]
    B = len(inputs["seq_length"])
    query = torch.cat([emb(c, inputs[c.name]).reshape(B, 1, -1) for c in sparse if c.name in history_feature_list],
                      -1)                                                                  # :68-69, 80
    keys = torch.cat([emb(c, inputs[c.name]) for c in hist], -1)                           # :70-71, 82
    deep = torch.cat([emb(c, inputs[c.name]).reshape(B, 1, -1) for c in sparse], -1)      # :72-73, 81
    T = keys.shape[1]
    ln = torch.as_tensor(inputs["seq_length"]).reshape(-1)
    valid = torch.arange(T)[None, :] < ln[:, None]
    out = keys
    for i in range(transformer_num):                                                       # :85-92
        out = transformer(out, out, valid, valid, W["transformers"][i], att_head_num, use_layer_norm=True,
                          blinding=False, output_type=None)
    att = O.attention_sequence_pooling(query, out, valid, W["lau"], att_activation="sigmoid",
                                       weight_normalization=True)                          # :94-96
    flat = torch.cat([deep, att], -1).flatten(1)                                           # :97-98
    dv = [torch.as_tensor(inputs[c.name], dtype=torch.float32).reshape(B, -1) for c in dense]
    x = torch.cat([flat] + dv, -1) if dv else flat                                         # :100
    h = O.dnn(x, W["dnn_kernels"], W["dnn_biases"], "relu")                                # :101
    logit = h @ W["dense_kernel"]                                                          # :102
    return logit, O.prediction(logit, W.get("global_bias"), task)                          # :103
