"""The golden checks, written once: the model-level ones for every fixture family of golden_models.FAMILIES, the
layer-level ones for every fixture set of golden_models.LAYER_SETS.

Each family's test modules bind them under their own test names, so adding a family or a layer set needs only its
record, its oracle functions and these bindings:

    T = model_golden_checks.model_tests("pairwise")          # CPU
    test_oracle_matches_reference_model = T.oracle
    T = model_golden_checks.gpu_model_tests("pairwise")      # GPU, both GEMM precisions
    test_model_forward_matches_reference = T.forward
    test_oracle_matches_reference_layer = model_golden_checks.layer_tests("pairwise").oracle
    test_layer_fixture = model_golden_checks.gpu_layer_test("pairwise")

Every call makes new function objects, so the marks of one module never reach another.

Layer fixtures (the reference's layer run on given inputs and weights, with the gradients for a seeded ``dout``):
on the CPU the set's restatement reproduces the output and every input and weight gradient (a gradient that is 0
comes out exactly 0); on the GPU, in both GEMM precisions, the deepctr_b200 layer built from the fixture's arguments,
with exactly the fixture's weight set loaded by name, reproduces the output and, run on a tape, every gradient.

Model fixtures, CPU, per fixture:
1. the family's restatement (oracle/models.py, tests/*_oracle.py) reproduces the logits, predictions, loss and
   every weight gradient;
2. the deepctr_b200 builders create exactly the reference's weight set (names, shapes, trainable flags, order) -
   the precondition for loading reference weights by name;
3. they build the graph the reference's builder SOURCE FILES build on this package (tests/golden/
   reference_builders*.json: inputs, layers, weights, planner slots) and have the reference's keyword defaults.
Model fixtures, GPU, per fixture, in both GEMM precisions (and with and without the DNN-input placement where the
family has it): the reference's weights loaded by name reproduce the logits and predictions (1e-4 relative), and one
SGD step's loss and weight updates  -lr * dL/dw  match the gradient torch autograd took THROUGH the reference's graph.
On synthetic Criteo-like data (b2_helpers.train): a graph-replayed training step equals an eager one, and the
DNN-input placement gives the unplaced results.
"""
import inspect
import types

import numpy as np
import pytest
import torch

import b2_helpers as H
import golden_models as G


# ---- CPU ----------------------------------------------------------------------------------------------
def check_fixture_set(fam):
    fxs = [fam.fixture(n) for n in fam.cases]
    assert len(fxs) == fam.n_cases
    assert {fx.builder for fx in fxs} == set(fam.builders)
    assert {fx.task for fx in fxs} == fam.tasks


def _close(got, want, rtol, atol, max_rel, what):
    """Within rtol / atol of each element, and within max_rel x the largest |want| overall."""
    got = np.asarray(got).reshape(want.shape)
    np.testing.assert_allclose(got, want, rtol=rtol, atol=atol, err_msg=what)
    err = float(np.abs(got - want).max())
    assert err <= max_rel * float(np.abs(want).max()), "%s: max error %.3e" % (what, err)


def check_oracle(fam, name):
    fx = fam.fixture(name)
    W, leaves = fam.oracle_weights(fx, requires_grad=True)
    logit, pred = fam.oracle_forward(fx, W)
    _close(logit.detach().numpy(), fx.logit, 1e-4, 1e-5, 1e-5, "logit")
    _close(pred.detach().numpy(), fx.out, 1e-4, 1e-6, 1e-5, "prediction")
    loss = G.loss_of(fx, pred)
    assert abs(float(loss.detach()) - fx.loss) <= 1e-5 * max(1.0, abs(fx.loss)), (float(loss), fx.loss)
    loss.backward()
    missing = set(k for k in fx.g if not G._ignored(k)) - set(leaves)
    assert not missing, "fixture gradients without an oracle leaf: %s" % sorted(missing)
    for key, want in fx.g.items():
        if G._ignored(key):
            assert not np.any(want), key           # the reference's discarded lookup pass gets no gradient
            continue
        leaf = leaves[key]
        got = leaf.grad.numpy() if leaf.grad is not None else np.zeros_like(want)
        _close(got, want, 1e-4, 1e-4 * float(np.abs(want).max()) + 1e-7, 1e-4, key)


def check_weight_set(fam, name):
    fx = fam.fixture(name)
    model = G.build(fx)
    wm = G.weight_map(fx, model)           # raises on any name / shape difference
    ref = [k for k in fx.w if not G._ignored(k)]
    assert len(wm) == len(ref)
    if name not in fam.graph_weight_order:
        key_of = {id(w): k for k, w in wm.items()}
        mine = [key_of[id(w)] for w in model.weights]
        assert mine == ref, "weight order: here %s, reference %s" % (mine, ref)
    # trainable flags: everything the reference differentiates is trainable here and vice versa
    for key, w in wm.items():
        assert w.trainable == (key in fx.g), key


def check_graph(fam, name):
    fx = fam.fixture(name)
    want = fam.reference_builders()["signatures"][name]
    model = G.build(fx)
    got = G.signature(model)
    assert want["inputs"] == got["inputs"], (want["inputs"], got["inputs"])
    assert want["weights"] == got["weights"], (want["weights"], got["weights"])
    assert want["slots"] == got["slots"] and want["fast"] == got["fast"]
    # the op graph: same multiset of (layer class, name); the topological order may differ where the
    # reference builds a branch earlier than it consumes it
    assert sorted(want["layers"]) == sorted(got["layers"]), (sorted(want["layers"]), sorted(got["layers"]))
    G.weight_map(fx, model)                # and the graph carries the reference-produced weights by name


def check_defaults(fam):
    """every keyword and default of the family's reference builders exists here with the same default."""
    from deepctr_b200 import models as M
    ref = fam.reference_builders()["defaults"]
    assert sorted(ref) == sorted(fam.builders)
    for b in fam.builders:
        mine = inspect.signature(getattr(M, b))
        assert [k for k, _ in ref[b]] == list(mine.parameters), b
        for k, d in ref[b]:
            assert d == repr(mine.parameters[k].default), (b, k, d, repr(mine.parameters[k].default))


def model_tests(family):
    """The CPU tests of one family: oracle, weight_set, graph (parametrised by fixture name), defaults and
    fixture_set."""
    fam = G.FAMILIES[family]
    cases = pytest.mark.parametrize("name", fam.cases)

    @cases
    def oracle(name):
        check_oracle(fam, name)

    @cases
    def weight_set(name):
        check_weight_set(fam, name)

    @cases
    def graph(name):
        check_graph(fam, name)

    def defaults():
        check_defaults(fam)

    def fixture_set():
        check_fixture_set(fam)
    return types.SimpleNamespace(oracle=oracle, weight_set=weight_set, graph=graph, defaults=defaults,
                                 fixture_set=fixture_set)


# ---- GPU ----------------------------------------------------------------------------------------------
@pytest.fixture(params=[True, False], ids=["placed", "unplaced"])
def placement(request):
    """DNN-input placement on / off while the model is built (for the families whose builders place their products
    in the DNN input)."""
    from deepctr_b200 import inputs as I
    I.DNN_INPUT_PLACEMENT = request.param
    yield request.param
    I.DNN_INPUT_PLACEMENT = True


def _model(fam, name):
    fx = fam.fixture(name)
    model = G.build(fx)
    return fx, model, G.assign_weights(fx, model)


def check_forward(fam, name):
    fx, model, _ = _model(fam, name)
    if fx.training and "dice" in name:       # predict() runs Dice on its moving statistics
        return
    x = fx.inputs()
    np.testing.assert_allclose(H.logits(model, x), fx.logit, rtol=1e-4, atol=H.logit_tol(fx.logit))
    atol = fam.predict_atol or H.logit_tol(fx.out)
    np.testing.assert_allclose(model.predict(x, batch_size=len(fx.y)), fx.out, rtol=1e-4, atol=atol)


def check_sgd_step(fam, name):
    from deepctr_b200.engine import SGD
    fx, model, wm = _model(fam, name)
    lr = 0.5
    model.compile(SGD(lr), "binary_crossentropy" if fx.task == "binary" else "mse", embedding_update="dense")
    loss = model.train_on_batch(fx.inputs(), fx.y)
    assert abs(loss - fx.loss) <= 2e-4 * max(1.0, abs(fx.loss)), (loss, fx.loss)
    for key, w in wm.items():
        if key not in fx.g:
            continue
        want = fx.g[key]
        got = (fx.w[key] - w.value()) / lr
        gmax = float(np.abs(want).max())
        np.testing.assert_allclose(got, want, rtol=2e-3, atol=3e-4 * gmax + 2e-6, err_msg=key)


def gpu_model_tests(family):
    """The GPU tests of one family, parametrised by fixture name and GEMM precision (and DNN-input placement where the
    family has it: a placed family's module imports ``placement`` from here): forward and sgd_step."""
    fam = G.FAMILIES[family]
    fixtures = ("gemm_precision", "placement") if fam.placed else ("gemm_precision",)

    def marks(f):
        return pytest.mark.gpu(pytest.mark.usefixtures(*fixtures)(pytest.mark.parametrize("name", fam.cases)(f)))

    @marks
    def forward(cuda, name):
        check_forward(fam, name)

    @marks
    def sgd_step(cuda, name):
        if "dice" in name and not fam.fixture(name).training:
            pytest.skip("fixture differentiates Dice in inference mode; a training step uses batch statistics")
        check_sgd_step(fam, name)
    return types.SimpleNamespace(forward=forward, sgd_step=sgd_step)


# ---- layer fixtures -----------------------------------------------------------------------------------
def check_layer_set(ls):
    assert len(ls.cases) == ls.n_cases
    assert {ls.load(n)[0]["layer"] for n in ls.cases} == set(ls.layers)


def _gradient_keys(d):
    return [k for k in d if k.startswith(("gx", "g_"))]


def check_layer_oracle(ls, name):
    meta, d = ls.load(name)
    keys = ["x"] if "x" in d else G.numbered(d, "x_")
    xs = {k: torch.tensor(d[k], requires_grad=d[k].dtype == np.float32) for k in keys}
    W = {k[2:]: torch.tensor(d[k], requires_grad=True) for k in d if k.startswith("w_")}
    out = ls.oracle(meta, list(xs.values()), W, d)
    out_close, grad_close = ls.cpu
    out_close(out.detach().numpy(), d["out"], "out")
    (out * torch.as_tensor(d["dout"])).sum().backward()
    leaves = {"g" + k: t for k, t in xs.items()}
    leaves.update(("g_" + k, t) for k, t in W.items())
    for key in _gradient_keys(d):
        want = d[key]
        got = leaves[key].grad.numpy() if leaves[key].grad is not None else np.zeros_like(want)
        if np.any(want):
            grad_close(got, want, key)
        else:
            np.testing.assert_array_equal(got, 0, err_msg=key)


def check_layer_gpu(ls, name, device):
    from deepctr_b200 import engine as E
    from deepctr_b200 import layers as LY
    meta, d = ls.load(name)
    kwargs = dict(meta["kwargs"])
    for k in ("layer_size", "att_hidden_units", "hidden_units"):
        if k in kwargs:
            kwargs[k] = tuple(kwargs[k])
    E.clear_session()
    layer = getattr(LY, meta["layer"])(**kwargs)
    arg, inputs = ls.args(meta, d, device)
    layer._maybe_build(E._shape_of(arg))
    mine = {w.name.split("/", 1)[1]: w for w in layer.weights}
    ref = {ls.weight_name(k[2:]): k[2:] for k in d if k.startswith("w_")}
    assert sorted(mine) == sorted(ref), (sorted(mine), sorted(ref))
    for n, w in mine.items():
        w.set_value(d["w_" + ref[n]])
    tape = E.Tape()
    with E.recording(tape):
        y = layer._invoke(arg, bool(meta.get("extra", {}).get("training", False)))
    # a list output (SENETLayer's F [B,1,E] windows) is compared and seeded field by field
    ys, part = (y, lambda a, i: a[:, i:i + 1]) if isinstance(y, list) else ([y], lambda a, i: a)
    out_close, grad_close = ls.gpu
    for i, yi in enumerate(ys):
        want = part(d["out"], i)
        out_close(E.contiguous(yi).cpu().numpy().reshape(want.shape), want, "out")
    if "dout" not in d:             # the root set holds outputs only
        return
    for i, yi in enumerate(ys):
        yi.requires_grad = True
        E.add_grad(yi, torch.tensor(part(d["dout"], i), device=device).reshape(yi.shape))
    tape.backward()
    leaves = {"g" + k: v for k, v in inputs.items()}
    leaves.update(("g_" + ref[n], w) for n, w in mine.items())
    for key in _gradient_keys(d):
        want = d[key]
        g = leaves[key].grad
        got = g.cpu().numpy().reshape(want.shape) if g is not None else np.zeros_like(want)
        grad_close(got, want, key)


def layer_tests(layer_set):
    """The CPU tests of one layer-fixture set: oracle (parametrised by fixture name) and fixture_set."""
    ls = G.LAYER_SETS[layer_set]

    @pytest.mark.parametrize("name", ls.cases)
    def oracle(name):
        check_layer_oracle(ls, name)

    def fixture_set():
        check_layer_set(ls)
    return types.SimpleNamespace(oracle=oracle, fixture_set=fixture_set)


def gpu_layer_test(layer_set):
    """The GPU test of one layer-fixture set, parametrised by fixture name and GEMM precision: the layer reproduces
    the output and, where the fixture has them, the input and weight gradients."""
    ls = G.LAYER_SETS[layer_set]

    @pytest.mark.gpu
    @pytest.mark.usefixtures("gemm_precision")
    @pytest.mark.parametrize("name", ls.cases)
    def layer(cuda, name):
        check_layer_gpu(ls, name, cuda)
    return layer


def graph_replay_test(cases):
    """A test over ``cases`` (builder, kw): six graph-replayed training steps equal six eager ones."""
    @pytest.mark.gpu
    @pytest.mark.parametrize("builder,kw", cases)
    def test(cuda, builder, kw):
        l_graph, w_graph, replayed, init = H.train(builder, "auto", kw)
        l_eager, w_eager, _, _ = H.train(builder, "off", kw, init=init)
        assert replayed > 0, "the training step was never replayed as a CUDA graph"
        np.testing.assert_allclose(l_graph, l_eager, rtol=1e-5, atol=1e-6)
        for k, v in w_eager.items():
            np.testing.assert_allclose(w_graph[k], v, rtol=1e-4, atol=1e-6 + 1e-4 * float(np.abs(v).max()),
                                       err_msg=k)
    return test


def placement_test(cases):
    """A test over ``cases`` (builder, kw, rtol, atol): six steps with the DNN-input placement give the unplaced
    results.  The same arithmetic on differently laid out operands (the unplaced DNN input is its own tensor, the
    placed one a window of the gather buffer) agrees to rounding, e.g. 5e-11 on an embedding of 1e-5; weights within
    rtol and atol x their largest value."""
    @pytest.mark.gpu
    @pytest.mark.parametrize("builder,kw,rtol,atol", cases)
    def test(cuda, builder, kw, rtol, atol):
        l_p, w_p, _, init = H.train(builder, "off", kw)
        l_u, w_u, _, _ = H.train(builder, "off", kw, placed=False, init=init)
        np.testing.assert_allclose(l_p, l_u, rtol=1e-6, atol=0)
        for k, v in w_u.items():
            np.testing.assert_allclose(w_p[k], v, rtol=rtol, atol=atol * float(np.abs(v).max()), err_msg=k)
    return test
