"""GPU parity of every hot-path operator layer (forward + gradients) against the CPU oracle.
Parametrisation follows the reference's own layer tests (tests/layers/interaction_test.py:11-126,
sequence_test.py:17-51, core_test.py:15-65, activations_test.py) with real numeric assertions added."""
import numpy as np
import pytest
import torch

from oracle import ops as O
import b2_helpers as H

pytestmark = [pytest.mark.gpu, pytest.mark.usefixtures("gemm_precision")]
RTOL, ATOL = 1e-4, 1e-5


def _run(layer, inputs, grad_out_rng, training=False):
    """Eager forward + backward of a layer.  Returns (output numpy, [input grads], {weight name: grad})."""
    from deepctr_b200 import engine as E
    vars_in = E._map_structure(E.to_var, inputs)
    for v in E._flatten(vars_in):
        if v.data.dtype == torch.float32:
            v.requires_grad = True
    tape = E.Tape()
    with E.recording(tape):
        layer._maybe_build(E._shape_of(vars_in))
        for w in layer.weights:
            w.materialize()
        y = layer._invoke(vars_in, training)
    out = E.contiguous(y).cpu().numpy()
    gy = grad_out_rng.normal(size=out.shape).astype(np.float32)
    y.requires_grad = True
    E.add_grad(y, torch.from_numpy(gy).to(y.data.device))
    tape.backward()
    gin = [v.grad.cpu().numpy().reshape(v.shape) if v.grad is not None else None for v in E._flatten(vars_in)]
    gw = {w.name.split("/", 1)[1]: (w.grad.cpu().numpy() if w.grad is not None else None) for w in layer.weights}
    return out, gy, gin, gw


def _t(a, grad=True):
    return torch.tensor(np.asarray(a), requires_grad=grad)


def _close(a, b, rtol=RTOL, atol=ATOL):
    a, b = np.asarray(a), np.asarray(b)
    from deepctr_b200 import ops, _lib as L
    if ops.GEMM_PRECISION == L.GEMM_BF16X3 and b.size:
        # split-bf16 GEMMs: the error is bounded relative to sum |a||b| of the dot product, not to the
        # (possibly cancelling) result -> normwise 1e-4 instead of elementwise
        atol = max(atol, 1e-4 * float(np.abs(b).max()))
    np.testing.assert_allclose(a, b, rtol=rtol, atol=atol)


def test_fm_layer(cuda):
    from deepctr_b200.layers import FM
    rng = np.random.RandomState(0)
    x = rng.normal(size=(5, 4, 3)).astype(np.float32)
    out, gy, gin, _ = _run(FM(), x, rng)
    xt = _t(x)
    want = O.fm(xt)
    (want * _t(gy, False)).sum().backward()
    _close(out, want.detach())
    _close(gin[0], xt.grad)
    with pytest.raises(ValueError):
        FM()(np.zeros((3, 4), np.float32))


@pytest.mark.parametrize("layer_num,param", [(0, "vector"), (1, "vector"), (3, "vector"), (2, "matrix")])
def test_crossnet(cuda, layer_num, param):
    from deepctr_b200.layers import CrossNet
    rng = np.random.RandomState(1)
    x = rng.normal(size=(33, 7)).astype(np.float32)
    layer = CrossNet(layer_num, parameterization=param)
    layer.build((None, 7))
    for w in layer.weights:
        w.set_value(rng.normal(0, 0.3, size=w.shape).astype(np.float32))
    out, gy, gin, gw = _run(layer, x, rng)
    xt = _t(x)
    ks = [_t(w.value()) for w in layer.kernels]
    bs = [_t(w.value()) for w in layer.bias]
    want = O.crossnet(xt, ks, bs, param)
    (want * _t(gy, False)).sum().backward()
    _close(out, want.detach())
    _close(gin[0], xt.grad)
    for i in range(layer_num):
        _close(gw["kernel%d" % i], ks[i].grad, 2e-4, 2e-5)
        _close(gw["bias%d" % i], bs[i].grad, 2e-4, 2e-5)
    with pytest.raises(ValueError):
        CrossNet(1)(np.zeros((2, 3, 4), np.float32))


@pytest.mark.parametrize("layer_size,split_half,act", [((10,), False, "relu"), ((10, 8), True, "relu"),
                                                       ((10, 8), False, "linear"), ((8, 6, 5), True, "sigmoid"),
                                                       ((128, 128), True, "relu")])
def test_cin(cuda, layer_size, split_half, act):
    from deepctr_b200.layers import CIN
    from deepctr_b200 import ops
    rng = np.random.RandomState(2)
    B, F, E_ = 37, 4, 3
    xstd, std = 1.0, 0.4
    if layer_size == (128, 128):
        # the C3 layer sizes at C3's 26 fields of 16: in fp32 precision the non-fused path, whose second layer
        # has h = 64 > 32 hidden maps (cin_outer_bwd's dense layout, two lane passes); inputs and weights scaled
        # so that the 676- and 1664-term contractions stay of order ten and the fp32 rounding of the CPU oracle
        # itself stays a tenth of the tolerance
        F, E_, xstd, std = 26, 16, 0.3, 0.1
    x = (xstd * rng.normal(size=(B, F, E_))).astype(np.float32)
    layer = CIN(layer_size, act, split_half, seed=3)
    layer.build((None, F, E_))
    for w in layer.weights:
        w.set_value(rng.normal(0, std, size=w.shape).astype(np.float32))
    old = ops.CIN_CHUNK_BYTES
    ops.CIN_CHUNK_BYTES = 4 * E_ * F * 10 * 11      # force several batch chunks
    try:
        out, gy, gin, gw = _run(layer, x, rng)
    finally:
        ops.CIN_CHUNK_BYTES = old
    xt = _t(x)
    fs = [_t(w.value()) for w in layer.filters]
    bs = [_t(w.value()) for w in layer.bias]
    want = O.cin(xt, fs, bs, layer_size, act, split_half)
    (want * _t(gy, False)).sum().backward()
    assert out.shape == tuple(want.shape)
    _close(out, want.detach())
    _close(gin[0], xt.grad, 3e-4, 3e-5)
    for i in range(len(layer_size)):
        _close(gw["filter%d" % i], fs[i].grad, 3e-4, 3e-5)
        _close(gw["bias%d" % i], bs[i].grad, 3e-4, 3e-5)
    # closed form of SURVEY.md 8c for the first layer: einsum('bid,bjd,ijn->bdn')
    W0 = fs[0].detach()[0].reshape(F, F, layer_size[0])
    y0 = torch.einsum("bid,bjd,ijn->bdn", xt.detach(), xt.detach(), W0) + bs[0].detach()
    if len(layer_size) == 1:
        _close(out, O._ACT[act](y0).sum(dim=1))
    with pytest.raises(ValueError):
        CIN((3, 4), split_half=True).build((None, 4, 3))   # odd hidden size with split_half


@pytest.mark.parametrize("heads,use_res,scaling", [(1, True, False), (2, False, False), (2, True, True)])
def test_interacting_layer(cuda, heads, use_res, scaling):
    from deepctr_b200.layers import InteractingLayer
    rng = np.random.RandomState(3)
    B, F, E_ = 21, 4, 3
    x = rng.normal(size=(B, F, E_)).astype(np.float32)
    layer = InteractingLayer(att_embedding_size=5, head_num=heads, use_res=use_res, scaling=scaling)
    layer.build((None, F, E_))
    for w in layer.weights:
        w.set_value(rng.normal(0, 0.5, size=w.shape).astype(np.float32))
    out, gy, gin, gw = _run(layer, x, rng)
    xt = _t(x)
    wq, wk, wv = _t(layer.W_Query.value()), _t(layer.W_key.value()), _t(layer.W_Value.value())
    wr = _t(layer.W_Res.value()) if use_res else None
    want = O.interacting(xt, wq, wk, wv, wr, heads, 5, use_res, scaling)
    (want * _t(gy, False)).sum().backward()
    _close(out, want.detach())
    _close(gin[0], xt.grad, 3e-4, 3e-5)
    _close(gw["query"], wq.grad, 3e-4, 3e-5)
    _close(gw["key"], wk.grad, 3e-4, 3e-5)
    _close(gw["value"], wv.grad, 3e-4, 3e-5)
    if use_res:
        _close(gw["res"], wr.grad, 3e-4, 3e-5)


@pytest.mark.parametrize("act", ["relu", "sigmoid", "dice"])
@pytest.mark.parametrize("training", [False, True])
def test_dnn_layer(cuda, act, training):
    from deepctr_b200.layers import DNN
    rng = np.random.RandomState(4)
    x = rng.normal(size=(65, 9)).astype(np.float32)
    layer = DNN((7, 5), activation=act, seed=1)
    layer.build((None, 9))
    H.randomize_weights(layer, rng, 0.4)
    out, gy, gin, gw = _run(layer, x, rng, training=training)
    xt = _t(x)
    ks = [_t(w.value()) for w in layer.kernels]
    bs = [_t(w.value()) for w in layer.bias]
    params = None
    if act == "dice":
        # moving statistics were already updated by the training forward: rebuild the pre-step values
        params = []
        for al in layer.activation_layers:
            params.append({"alphas": _t(al.alphas.value()), "moving_mean": _t(al.moving_mean.value(), False),
                           "moving_var": _t(al.moving_variance.value(), False)})
        if training:
            for p in params:       # batch statistics are used in training: moving values are irrelevant
                p["moving_mean"], p["moving_var"] = None, None
    want = O.dnn(xt, ks, bs, act, None, params, training)
    (want * _t(gy, False)).sum().backward()
    _close(out, want.detach(), 2e-4, 2e-5)
    _close(gin[0], xt.grad, 5e-4, 5e-5)
    for i in range(2):
        _close(gw["kernel%d" % i], ks[i].grad, 5e-4, 5e-5)
        _close(gw["bias%d" % i], bs[i].grad, 5e-4, 5e-5)
    if act == "dice":
        for i, p in enumerate(params):
            _close(gw["act%d/dice_alpha" % i] if ("act%d/dice_alpha" % i) in gw else
                   [v for k, v in gw.items() if k.endswith("act%d/dice_alpha" % i)][0], p["alphas"].grad, 5e-4, 5e-5)


def test_dice_moving_statistics_update(cuda):
    from deepctr_b200.layers import Dice
    rng = np.random.RandomState(5)
    x = (rng.normal(size=(200, 3)) * 2 + 1).astype(np.float32)
    layer = Dice()
    layer.build((None, 3))
    _run(layer, x, rng, training=True)
    np.testing.assert_allclose(layer.moving_mean.value(), 0.01 * x.mean(0), rtol=1e-4, atol=1e-6)
    np.testing.assert_allclose(layer.moving_variance.value(), 0.99 + 0.01 * x.var(0), rtol=1e-4, atol=1e-6)


@pytest.mark.parametrize("mode", ["sum", "mean", "max"])
@pytest.mark.parametrize("masking", [False, True])
def test_sequence_pooling_layer_standalone(cuda, mode, masking):
    from deepctr_b200.layers import SequencePoolingLayer
    from deepctr_b200 import engine as E
    rng = np.random.RandomState(6)
    B, T, E_ = 4, 10, 8
    x = rng.normal(size=(B, T, E_)).astype(np.float32)
    lens = np.array([[0], [3], [10], [7]], dtype=np.int32)
    layer = SequencePoolingLayer(mode, supports_masking=masking)
    if masking:
        ids = (np.arange(T)[None, :] < lens).astype(np.int32)
        xv = E.to_var(x)
        xv.mask = E.KMask(ids=[torch.from_numpy(ids).to(xv.data.device)])
        out, gy, gin, _ = _run(layer, xv, rng)
        want_in = dict(mask=torch.from_numpy(ids) != 0)
    else:
        out, gy, gin, _ = _run(layer, [x, lens], rng)
        want_in = dict(lengths=torch.from_numpy(lens.reshape(-1)))
    xt = _t(x)
    want = O.sequence_pooling(xt, mode, **want_in)
    (want * _t(gy, False)).sum().backward()
    assert np.array_equal(out, want.detach().numpy()), "pooled sums are bit-exact"
    _close(gin[0], xt.grad)


@pytest.mark.parametrize("norm", [True, False])
def test_weighted_sequence_layer_standalone(cuda, norm):
    from deepctr_b200.layers import WeightedSequenceLayer
    rng = np.random.RandomState(7)
    B, T, E_ = 6, 5, 4
    x = rng.normal(size=(B, T, E_)).astype(np.float32)
    w = rng.rand(B, T, 1).astype(np.float32)
    lens = rng.randint(1, T + 1, size=(B, 1)).astype(np.int32)
    out, gy, gin, _ = _run(WeightedSequenceLayer(norm), [x, lens, w], rng)
    xt = _t(x)
    want = O.weighted_sequence(xt, torch.from_numpy(w), norm, lengths=torch.from_numpy(lens.reshape(-1)))
    (want * _t(gy, False)).sum().backward()
    _close(out, want.detach(), 1e-5, 1e-6)
    _close(gin[0], xt.grad, 1e-5, 1e-6)


@pytest.mark.parametrize("weight_normalization", [False, True])
@pytest.mark.parametrize("act", ["sigmoid", "dice"])
def test_attention_sequence_pooling_layer(cuda, weight_normalization, act):
    from deepctr_b200.layers import AttentionSequencePoolingLayer
    rng = np.random.RandomState(8)
    B, T, E_ = 4, 10, 8
    q = rng.normal(size=(B, 1, E_)).astype(np.float32)
    k = rng.normal(size=(B, T, E_)).astype(np.float32)
    lens = np.array([[1], [10], [4], [7]], dtype=np.int32)
    layer = AttentionSequencePoolingLayer((6, 5), act, weight_normalization=weight_normalization)
    layer.build([(None, 1, E_), (None, T, E_), (None, 1)])
    H.randomize_weights(layer, rng, 0.4)
    out, gy, gin, gw = _run(layer, [q, k, lens], rng)
    qt, kt = _t(q), _t(k)
    lau = layer.local_att
    W = {"dnn_kernels": [_t(w.value()) for w in lau.dnn.kernels], "dnn_biases": [_t(w.value()) for w in lau.dnn.bias],
         "kernel": _t(lau.kernel.value()), "bias": _t(lau.bias.value())}
    if act == "dice":
        W["act_params"] = [{"alphas": _t(al.alphas.value()), "moving_mean": _t(al.moving_mean.value(), False),
                            "moving_var": _t(al.moving_variance.value(), False)} for al in lau.dnn.activation_layers]
    mask = O.sequence_mask(torch.from_numpy(lens.reshape(-1)), T)
    want = O.attention_sequence_pooling(qt, kt, mask, W, act, weight_normalization)
    (want * _t(gy, False)).sum().backward()
    assert out.shape == (B, 1, E_)
    _close(out, want.detach(), 2e-4, 2e-5)
    _close(gin[0], qt.grad, 5e-4, 5e-5)
    _close(gin[1], kt.grad, 5e-4, 5e-5)
    _close([v for n, v in gw.items() if n.endswith("local_activation_unit/kernel")][0], W["kernel"].grad, 5e-4, 5e-5)
    for i in range(2):
        _close([v for n, v in gw.items() if n.endswith("dnn/kernel%d" % i)][0], W["dnn_kernels"][i].grad, 5e-4, 5e-5)
    # padded positions receive exactly zero gradient (Appendix F.6)
    for b in range(B):
        assert np.all(gin[1][b, lens[b, 0]:] == 0)


def test_prediction_and_linear_layers(cuda):
    from deepctr_b200.layers import PredictionLayer, Linear
    rng = np.random.RandomState(9)
    z = rng.normal(size=(50, 1)).astype(np.float32)
    for task in ["binary", "regression"]:
        layer = PredictionLayer(task)
        layer.build((None, 1))
        layer.global_bias.set_value(np.array([0.25], np.float32))
        got = layer(z)
        want = O.prediction(torch.from_numpy(z), torch.tensor([0.25]), task)
        _close(got.data.cpu().numpy(), want.numpy(), 1e-5, 1e-6)
    with pytest.raises(ValueError):
        PredictionLayer("ranking")
    with pytest.raises(ValueError):
        Linear(mode=3)
    sp = rng.normal(size=(20, 1, 6)).astype(np.float32)
    dn = rng.normal(size=(20, 4)).astype(np.float32)
    lin = Linear(mode=2, use_bias=True)
    lin.build([(None, 1, 6), (None, 4)])
    lin.kernel.set_value(rng.normal(size=(4, 1)).astype(np.float32))
    lin.bias.set_value(np.array([0.5], np.float32))
    got = lin([sp, dn]).data.cpu().numpy()
    want = O.linear(torch.from_numpy(sp), torch.from_numpy(dn), torch.from_numpy(lin.kernel.value()),
                    torch.tensor([0.5]))
    _close(got, want.numpy())
    # mode 0 (sparse part only) with a bias: rowsum + scalar bias, gradients to the input and to the bias
    lin0 = Linear(mode=0, use_bias=True)
    lin0.build((None, 1, 6))
    lin0.bias.set_value(np.array([-0.75], np.float32))
    out, gy, gin, gw = _run(lin0, sp, rng, training=True)
    _close(out, sp.sum(-1) - 0.75)
    _close(gin[0], np.broadcast_to(gy.reshape(20, 1, 1), sp.shape))
    _close([v for n, v in gw.items() if n.endswith("linear_bias")][0], gy.sum().reshape(1), 1e-4, 1e-5)


def test_hash_layer_device_and_vocabulary(cuda, tmp_path):
    from deepctr_b200.layers import Hash
    ids = np.array([[0], [1], [12345], [99999999]], dtype=np.int32)
    for mz in (False, True):
        got = Hash(100, mask_zero=mz)(ids).data.cpu().numpy()
        assert np.array_equal(got, O.hash_layer(ids, 100, mz))
    # the reference's only known-answer vector (tests/layers/utils_test.py:20-22)
    p = tmp_path / "vocab.csv"
    p.write_text("1,lake\n2,merson\n3,johnson\n")
    out = Hash(num_buckets=4, vocabulary_path=str(p))([["lake"], ["johnson"], ["lakemerson"]])
    assert np.array_equal(np.asarray(out), [[1], [3], [0]])


@pytest.mark.parametrize("training", [False, True])
def test_dnn_with_batchnorm(cuda, training):
    """DNN(use_bn=True): tensordot + bias -> BatchNormalization -> activation (layers/core.py:193-200)."""
    from deepctr_b200.layers import DNN
    rng = np.random.RandomState(31)
    x = rng.normal(size=(77, 6)).astype(np.float32)
    layer = DNN((5, 4), activation="relu", use_bn=True, seed=2)
    layer.build((None, 6))
    H.randomize_weights(layer, rng, 0.5)
    bn_before = [{"gamma": _t(b.gamma.value()), "beta": _t(b.beta.value()),
                  "moving_mean": _t(b.moving_mean.value(), False), "moving_var": _t(b.moving_variance.value(), False)}
                 for b in layer.bn_layers]
    out, gy, gin, gw = _run(layer, x, rng, training=training)
    xt = _t(x)
    ks = [_t(w.value()) for w in layer.kernels]
    bs = [_t(w.value()) for w in layer.bias]
    want = O.dnn(xt, ks, bs, "relu", None, None, training, bn_params=bn_before)
    (want * _t(gy, False)).sum().backward()
    _close(out, want.detach(), 3e-4, 3e-5)
    _close(gin[0], xt.grad, 1e-3, 1e-4)
    for i in range(2):
        _close(gw["kernel%d" % i], ks[i].grad, 1e-3, 1e-4)
        _close(gw["bn%d/gamma" % i], bn_before[i]["gamma"].grad, 1e-3, 1e-4)
        _close(gw["bn%d/beta" % i], bn_before[i]["beta"].grad, 1e-3, 1e-4)
    if training:   # moving statistics moved towards the batch statistics with momentum 0.99
        h0 = (xt.detach() @ ks[0].detach() + bs[0].detach())
        np.testing.assert_allclose(layer.bn_layers[0].moving_mean.value(),
                                   0.99 * bn_before[0]["moving_mean"].numpy() + 0.01 * h0.mean(0).numpy(),
                                   rtol=1e-4, atol=1e-5)


def test_dropout_mask_is_consistent_between_forward_and_backward(cuda):
    from deepctr_b200 import engine as E, ops
    rng = np.random.RandomState(32)
    x = E.to_var(np.ones((4096, 16), np.float32))
    x.requires_grad = True
    tape = E.Tape()
    with E.recording(tape):
        y = ops.dropout(x, 0.25, seed=7)
    yv = y.data.cpu().numpy()
    kept = yv != 0
    assert abs(kept.mean() - 0.75) < 0.02
    np.testing.assert_allclose(yv[kept], 1.0 / 0.75, rtol=1e-6)
    E.add_grad(y, torch.ones_like(y.data))
    tape.backward()
    g = x.grad.cpu().numpy()
    assert np.array_equal(g != 0, kept) and np.allclose(g[kept], 1.0 / 0.75)
    # inference: identity
    from deepctr_b200.layers import DNN
    layer = DNN((8,), dropout_rate=0.5)
    a = layer(np.ones((10, 4), np.float32)).data.cpu().numpy()
    b = layer(np.ones((10, 4), np.float32)).data.cpu().numpy()
    assert np.array_equal(a, b)


@pytest.mark.parametrize("B,F,E_,layer_size,split_half,act", [
    (64, 6, 8, (40, 24), True, "relu"),          # h = 6 -> hp 32, h = 20 -> hp 32
    (64, 6, 8, (40, 24), False, "linear"),       # h = 40 -> hp 64
    (24, 5, 16, (136, 16), True, "relu"),        # h = 68 -> hp 128 (two k-blocks per i), N = 136 -> two N tiles? (bn 256)
    (300, 26, 16, (128, 128), True, "relu"),     # the C3 layer sizes: K' = 832 / 1664, 2-CTA tiles, ragged last row tile
])
@pytest.mark.parametrize("fold", [True, False])
def test_cin_fused_generated_outer_product(cuda, B, F, E_, layer_size, split_half, act, fold):
    """b2ctr_cin_gemm: the outer product is generated inside the tensor-core GEMM producer (forward and filter
    gradient); checked against the oracle's literal op sequence, all gradients."""
    from deepctr_b200.layers import CIN
    from deepctr_b200 import ops, _lib as L
    ops.set_gemm_precision("bf16x3")
    rng = np.random.RandomState(21)
    x = rng.normal(0, 0.5, size=(B, F, E_)).astype(np.float32)
    assert ops.cin_fusable(x, layer_size, split_half)
    layer = CIN(layer_size, act, split_half, seed=3)
    layer.build((None, F, E_))
    for w in layer.weights:
        w.set_value(rng.normal(0, 0.2, size=w.shape).astype(np.float32))
    L.reset_launch_count()
    old = ops.CIN_DZ_CHUNK_BYTES, ops.CIN_FOLD
    ops.CIN_DZ_CHUNK_BYTES = 4 * 832 * 1024          # several dZ row chunks at the larger shapes
    ops.CIN_FOLD = fold                               # dZ folded inside the GEMM epilogue / by a second kernel
    try:
        out, gy, gin, gw = _run(layer, x, rng)
    finally:
        ops.CIN_DZ_CHUNK_BYTES, ops.CIN_FOLD = old
    xt = _t(x)
    fs = [_t(w.value()) for w in layer.filters]
    bs = [_t(w.value()) for w in layer.bias]
    want = O.cin(xt, fs, bs, layer_size, act, split_half)
    (want * _t(gy, False)).sum().backward()

    def close(a, b, what):
        b = b.detach().numpy() if hasattr(b, "detach") else np.asarray(b)
        a = np.asarray(a)
        np.testing.assert_allclose(a.reshape(b.shape), b, rtol=2e-4, atol=2e-4 * float(np.abs(b).max()), err_msg=what)
    close(out, want, "out")
    close(gin[0], xt.grad, "dx")
    for i in range(len(layer_size)):
        close(gw["filter%d" % i], fs[i].grad, "filter%d" % i)
        close(gw["bias%d" % i], bs[i].grad, "bias%d" % i)


@pytest.mark.parametrize("B,T,E_,n,act", [(16, 20, 16, 24, "relu"), (40, 50, 64, 80, "sigmoid"), (9, 31, 8, 36, None)])
def test_din_first_attention_layer_generated_input(cuda, B, T, E_, n, act):
    """b2ctr_att_gemm: act([q, k, q-k, q*k] W + b) with the [B,T,4E] input generated inside the GEMM producer,
    forward + every gradient against torch."""
    from deepctr_b200 import engine as E, ops
    ops.set_gemm_precision("bf16x3")
    rng = np.random.RandomState(23)
    q = rng.normal(0, 0.5, size=(B, 1, E_)).astype(np.float32)
    k = rng.normal(0, 0.5, size=(B, T, E_)).astype(np.float32)
    w = rng.normal(0, 0.2, size=(4 * E_, n)).astype(np.float32)
    b = rng.normal(0, 0.2, size=(n,)).astype(np.float32)
    gy = rng.normal(size=(B, T, n)).astype(np.float32)
    qv, kv = E.to_var(q), E.to_var(k)
    wv, bv = E.to_var(w), E.to_var(b)
    for v in (qv, kv, wv, bv):
        v.requires_grad = True
    assert ops.din_att_fusable(qv, kv, n)
    tape = E.Tape()
    with E.recording(tape):
        y = ops.din_att_first(qv, kv, wv, bv, act)
    out = E.contiguous(y).cpu().numpy()
    y.requires_grad = True
    E.add_grad(y, torch.from_numpy(gy).to(y.data.device))
    tape.backward()
    qt, kt, wt, bt = _t(q), _t(k), _t(w), _t(b)
    qq = qt.expand(B, T, E_)
    a = torch.cat([qq, kt, qq - kt, qq * kt], dim=-1)
    want = a @ wt + bt
    want = {"sigmoid": torch.sigmoid, "relu": torch.relu, None: lambda v: v}[act](want)
    (want * torch.from_numpy(gy)).sum().backward()

    def close(got, ref, what):
        ref = ref.detach().numpy()
        np.testing.assert_allclose(np.asarray(got).reshape(ref.shape), ref, rtol=2e-4,
                                   atol=2e-4 * float(np.abs(ref).max()), err_msg=what)
    close(out, want, "out")
    close(qv.grad.cpu().numpy(), qt.grad, "dq")
    close(kv.grad.cpu().numpy(), kt.grad, "dk")
    close(wv.grad.cpu().numpy(), wt.grad, "dw")
    close(bv.grad.cpu().numpy(), bt.grad, "db")
