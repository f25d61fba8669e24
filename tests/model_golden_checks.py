"""The model-golden checks, written once for every fixture family of golden_models.FAMILIES.

Each family's test modules bind them under their own test names, so adding a family needs only its record in
FAMILIES, its oracle functions and these bindings:

    T = model_golden_checks.model_tests("pairwise")          # CPU
    test_oracle_matches_reference_model = T.oracle
    T = model_golden_checks.gpu_model_tests("pairwise")      # GPU, both GEMM precisions
    test_model_forward_matches_reference = T.forward

Every call makes new function objects, so the marks of one module never reach another.

CPU, per fixture:
1. the family's restatement (oracle/models.py, tests/*_oracle.py) reproduces the logits, predictions, loss and
   every weight gradient;
2. the deepctr_b200 builders create exactly the reference's weight set (names, shapes, trainable flags, order) -
   the precondition for loading reference weights by name;
3. they build the graph the reference's builder SOURCE FILES build on this package (tests/golden/
   reference_builders*.json: inputs, layers, weights, planner slots) and have the reference's keyword defaults.
GPU, per fixture, in both GEMM precisions (and with and without the DNN-input placement where the family has it):
the reference's weights loaded by name reproduce the logits and predictions (1e-4 relative), and one SGD step's
loss and weight updates  -lr * dL/dw  match the gradient torch autograd took THROUGH the reference's graph.
On synthetic Criteo-like data (b2_helpers.train): a graph-replayed training step equals an eager one, and the
DNN-input placement gives the unplaced results.
"""
import inspect
import types

import numpy as np
import pytest

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
