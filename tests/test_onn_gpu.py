"""GPU: the field-aware product kernels of ONN and the ONN builder.

* b2ctr_ffm_product_fwd / _bwd against float64 in both modes (elementwise and reduce_sum), over F = 2 / 7 / 26 and
  E = 4 / 8 (and E = 5, the scalar path), with single-valued fields and pre-pooled operands, the output a window of
  a wider buffer, and at the bench shape (26 fields x 1M ids, E = 4) with a reduced batch;
* the backward (the scratch pass) is bit-identical from run to run;
* out-of-range ids read zero rows and are counted; a model step raises ValueError and leaves the field's tables
  untouched;
* the forward allocates no [B, F(F-1), E] block;
* the 'sparse' SGD update equals -lr x the 'dense' gradient from the same weights on a batch with many repeated ids,
  so no sample's update is read by another sample's gradient.
Model fixtures (with model_golden_checks): logits and one SGD step in both GEMM precisions; a graph-replayed ONN step
equals an eager one.
"""
import itertools

import numpy as np
import pytest
import torch

import b2_helpers as H
import model_golden_checks as C
import onn_family  # noqa: F401  (registers the "onn" fixture family)

pytestmark = pytest.mark.gpu

T = C.gpu_model_tests("onn")
test_model_forward_matches_reference = T.forward
test_model_sgd_step_matches_reference_gradients = T.sgd_step
test_graph_replayed_step_equals_eager = C.graph_replay_test([
    pytest.param("ONN", dict(dnn_hidden_units=(32, 16)), id="onn"),
    pytest.param("ONN", dict(dnn_hidden_units=(16,), reduce_sum=True, use_bn=False), id="onn_reduce_sum")])


def _problem(cuda, B, F, E, V, seed, pooled=(), id_dtype=torch.int32):
    """Tables [V, E] for every (field, partner), ids [B] per single-valued field, a random [B, (F-1)*E] operand per
    pooled field (a window at column 4 of a wider buffer)."""
    from deepctr_b200 import kernels as K
    g = torch.Generator(device=cuda).manual_seed(seed)
    tables = [None] * (F * F)
    for a in range(F):
        for b in range(F):
            if a != b:
                tables[a * F + b] = torch.randn((V, E), generator=g, device=cuda) * 0.5
    ptrs = torch.tensor([t.data_ptr() if t is not None else 0 for t in tables], dtype=torch.int64, device=cuda)
    ids, ops_ = [], []
    for a in range(F):
        if a in pooled:
            w = torch.randn((B, (F - 1) * E + 8), generator=g, device=cuda)
            ops_.append(w[:, 4:4 + (F - 1) * E])
            ids.append(None)
        else:
            ids.append(torch.randint(0, V, (B,), generator=g, device=cuda, dtype=torch.int64).to(id_dtype))
            ops_.append(None)
    return tables, ptrs, ids, ops_, K


def _operand64(tables, ids, ops_, F, a, b):
    if ids[a] is None:
        s = b - (b > a)
        E = ops_[a].shape[1] // (F - 1)
        return ops_[a][:, s * E:(s + 1) * E].double().cpu()
    return tables[a * F + b].double().cpu()[ids[a].long().cpu()]


def _fields(K, ids, ops_, V, grads=None):
    return [K.ffm_field(idx=i, vocab=V, pooled=o, grad=grads[a] if grads is not None else None)
            for a, (i, o) in enumerate(zip(ids, ops_))]


def _check(cuda, B, F, E, V, reduce_sum, pooled=(), seed=0, rtol=1e-5):
    tables, ptrs, ids, ops_, K = _problem(cuda, B, F, E, V, seed, pooled)
    P = F * (F - 1) // 2
    w = P if reduce_sum else P * E
    out = torch.full((B, w + 12), 7.0, device=cuda)
    K.ffm_product_fwd(_fields(K, ids, ops_, V), ptrs, E, reduce_sum, out, 4, B)
    want = []
    for i, j in itertools.combinations(range(F), 2):
        p = _operand64(tables, ids, ops_, F, i, j) * _operand64(tables, ids, ops_, F, j, i)
        want.append(p.sum(-1, keepdim=True) if reduce_sum else p)
    want = torch.cat(want, 1)
    got = out.cpu()
    np.testing.assert_allclose(got[:, 4:4 + w].double().numpy(), want.numpy(), rtol=rtol, atol=1e-6)
    assert bool((got[:, :4] == 7).all()) and bool((got[:, 4 + w:] == 7).all())      # nothing outside the window
    # backward: per-lookup gradient rows into each field's slot of a [B, F(F-1)E] scratch
    dout = torch.randn((B, w + 12), device=cuda)
    scratch = torch.full((B, F * (F - 1) * E), 3.0, device=cuda)
    grads = [scratch[:, a * (F - 1) * E:] for a in range(F)]
    K.ffm_product_bwd(_fields(K, ids, ops_, V, grads), ptrs, E, reduce_sum, dout, 4, B)
    g64 = dout[:, 4:4 + w].double().cpu()
    want_rows = torch.zeros((B, F * (F - 1) * E), dtype=torch.float64)
    for p, (i, j) in enumerate(itertools.combinations(range(F), 2)):
        gp = g64[:, p:p + 1] if reduce_sum else g64[:, p * E:(p + 1) * E]
        ei, ej = _operand64(tables, ids, ops_, F, i, j), _operand64(tables, ids, ops_, F, j, i)
        ci, cj = (i * (F - 1) + j - 1) * E, (j * (F - 1) + i) * E
        want_rows[:, ci:ci + E] = gp * ej
        want_rows[:, cj:cj + E] = gp * ei
    np.testing.assert_allclose(scratch.cpu().double().numpy(), want_rows.numpy(), rtol=rtol, atol=1e-6)
    again = torch.empty_like(scratch)
    grads2 = [again[:, a * (F - 1) * E:] for a in range(F)]
    K.ffm_product_bwd(_fields(K, ids, ops_, V, grads2), ptrs, E, reduce_sum, dout, 4, B)
    assert torch.equal(scratch, again)                  # one writer per element: deterministic


@pytest.mark.parametrize("reduce_sum", [False, True], ids=["elementwise", "reduce_sum"])
@pytest.mark.parametrize("F,E", [(2, 4), (7, 8), (26, 4), (7, 5)])
@pytest.mark.parametrize("pooled", [(), (0, 3)], ids=["single", "pooled"])
def test_ffm_product_matches_float64(cuda, F, E, reduce_sum, pooled):
    pooled = tuple(a for a in pooled if a < F)
    _check(cuda, 515, F, E, 97, reduce_sum, pooled, seed=F * 10 + E)


@pytest.mark.parametrize("reduce_sum", [False, True], ids=["elementwise", "reduce_sum"])
def test_ffm_product_bench_shape(cuda, reduce_sum):
    """26 fields x 1M ids x E = 4 (650 tables, 10.4 GB), B = 2048."""
    _check(cuda, 2048, 26, 4, 1 << 20, reduce_sum, seed=3)


def test_out_of_range_ids_read_zero_rows_and_are_counted(cuda):
    from deepctr_b200 import kernels as K
    B, F, E, V = 64, 3, 4, 10
    tables, ptrs, ids, ops_, _ = _problem(cuda, B, F, E, V, 1)
    ids[0][::2] = V + 5
    ids[0][1::4] = -1
    K.embed_oob_count(reset=True)
    out = torch.empty((B, 3 * E), device=cuda)
    K.ffm_product_fwd(_fields(K, ids, ops_, V), ptrs, E, False, out, 0, B)
    bad = (ids[0] < 0) | (ids[0] >= V)
    assert K.embed_oob_count(reset=True) == int(bad.sum())
    # pairs (0, 1) and (0, 2) read a zero row for field 0
    assert bool((out[bad][:, :2 * E] == 0).all()) and bool((out[~bad][:, :2 * E] != 0).any())


def _onn_model(rng, n=256, F=6, V=40, E=4, **kw):
    from deepctr_b200 import engine as E_, models as M
    from deepctr_b200.feature_column import SparseFeat, DenseFeat
    cols = [SparseFeat("C%d" % i, V, E) for i in range(F)] + [DenseFeat("I0", 1)]
    x = {"C%d" % i: rng.randint(0, V, size=n).astype(np.int32) for i in range(F)}
    x["I0"] = rng.rand(n).astype(np.float32)
    y = (rng.rand(n) < 0.3).astype(np.float32)
    E_.clear_session()
    model = M.ONN(cols, cols, l2_reg_embedding=0, l2_reg_linear=0, **kw)
    return model, x, y


def test_out_of_range_ids_raise_and_update_nothing(cuda):
    from deepctr_b200.engine import SGD
    model, x, y = _onn_model(np.random.RandomState(2), dnn_hidden_units=(8,))
    model.compile(SGD(0.1), "binary_crossentropy", embedding_update="sparse", step_graph="off")
    x["C0"] = x["C0"] + 1000                            # every id of field 0 is out of range
    before = {t.embeddings.name: t.embeddings.value() for _, t in model.planner.ffm.tables}
    with pytest.raises(ValueError, match="outside"):
        model.train_on_batch(x, y)
    for _, t in model.planner.ffm.tables:
        if t.embeddings.name.startswith("sparse_emb_C0_"):
            np.testing.assert_array_equal(t.embeddings.value(), before[t.embeddings.name])
        elif "_C0/" in t.embeddings.name:                # partners see a zero row: a zero gradient
            np.testing.assert_array_equal(t.embeddings.value(), before[t.embeddings.name])


def test_forward_allocates_no_lookup_block(cuda, monkeypatch):
    """The [B, F(F-1), E] lookups never exist: no tensor the forward allocates holds as many elements.  The largest
    are the [B, P*E] products and what reads them (BatchNormalization, the DNN input), half that size."""
    model, x, _ = _onn_model(np.random.RandomState(3), n=8192, F=16, V=1000, dnn_hidden_units=(8,))
    model.predict(x, batch_size=8192)                   # warm up: tables, staging buffers
    sizes = []
    real_empty = torch.empty

    def empty_spy(*shape, **kw):
        t = real_empty(*shape, **kw)
        sizes.append(t.numel())
        return t
    monkeypatch.setattr(torch, "empty", empty_spy)
    model.predict(x, batch_size=8192)
    monkeypatch.setattr(torch, "empty", real_empty)
    assert sizes and max(sizes) < 8192 * 16 * 15 * 4
    assert 8192 * 120 * 4 in sizes                      # the products buffer: B x P*E


@pytest.mark.parametrize("reduce_sum", [False, True], ids=["elementwise", "reduce_sum"])
def test_sparse_update_equals_dense_gradient_with_repeated_ids(cuda, reduce_sum):
    """Many samples share each row (vocabulary 5, 1024 samples): the fused row-wise SGD update must be -lr x the dense
    gradient taken at the same pre-step weights."""
    from deepctr_b200.engine import SGD
    lr = 0.05
    res = {}
    init = None
    for mode in ("dense", "sparse"):
        model, x, y = _onn_model(np.random.RandomState(7), n=1024, F=5, V=5, dnn_hidden_units=(8,),
                                 reduce_sum=reduce_sum, use_bn=False)
        if init is None:
            init = [w.value() for w in model.weights]
        else:
            model.set_weights(init)
        model.compile(SGD(lr), "binary_crossentropy", embedding_update=mode, step_graph="off")
        model.train_on_batch(x, y)
        res[mode] = {t.embeddings.name: t.embeddings.value() for _, t in model.planner.ffm.tables}
    w0 = dict(zip([w.name for w in model.weights], init))
    for k in res["dense"]:
        d_dense = res["dense"][k] - w0[k]
        d_sparse = res["sparse"][k] - w0[k]
        np.testing.assert_allclose(d_sparse, d_dense, rtol=1e-4, atol=1e-6 * max(1.0, float(np.abs(d_dense).max())),
                                   err_msg=k)
        assert np.abs(d_dense).max() > 0, k
