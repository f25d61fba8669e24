"""CPU: the builders build what the reference's own builders build.

tests/golden/reference_builders.json records the graphs the reference's five builder SOURCE FILES build when
they are executed unmodified on this package (tests/golden/generate_builders.py): inputs, layer sequence
(class + Keras-style name), weights (name + shape + trainable), planner slots (i.e. the same single fused
gather launch), and every builder keyword with its default.  deepctr_b200.models must build the same graphs
for the same columns.  Graph construction needs no GPU.
"""
import json
import os

import pytest

import golden_models as G

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_builders.json")
BUILDERS = ("DeepFM", "xDeepFM", "DCN", "AutoInt", "DIN")


def signature(model):
    from deepctr_b200 import engine as E
    layers = [(type(l).__name__, l.name) for l in model.layers if not isinstance(l, E.InputLayer)]
    weights = [(w.name, tuple(w.shape), w.trainable) for w in model.weights]
    slots = [(s.emb.name, s.input_name, s.maxlen, s.pool, s.mask_mode, s.len_name, s.weight_name, s.weight_mode,
              s.dim, s.buf, s.col) for s in model.planner.slots]
    sig = {"inputs": list(model.input_names), "layers": layers, "weights": weights, "slots": slots,
           "fast": (model.planner.fast, getattr(model.planner, "fast_n", 0))}
    return json.loads(json.dumps(sig))      # tuples -> lists, as stored


def builder_args(fx):
    from deepctr_b200 import feature_column as FC
    kw = dict(fx.kwargs)
    for k in ("dnn_hidden_units", "cin_layer_size", "att_hidden_size", "fm_group"):
        if k in kw:
            kw[k] = tuple(kw[k])
    lin, dnn = G.columns(fx, "linear", FC), G.columns(fx, "dnn", FC)
    if fx.builder == "DIN":
        return (dnn, ["item_id", "cate_id"]), kw
    return (lin, dnn), kw


def _golden():
    with open(GOLDEN) as f:
        return json.load(f)


@pytest.mark.parametrize("name", G.CASES)
def test_reference_builder_source_runs_on_this_package(name):
    from deepctr_b200 import engine as E
    from deepctr_b200 import models as M
    fx = G.Fixture(name)
    args, kw = builder_args(fx)
    a = _golden()["signatures"][name]
    E.clear_session()
    ours = getattr(M, fx.builder)(*args, **kw)
    b = signature(ours)
    assert a["inputs"] == b["inputs"]
    assert a["weights"] == b["weights"]
    assert a["slots"] == b["slots"] and a["fast"] == b["fast"]
    # the op graph: same multiset of (layer class, name); the topological order may differ where the
    # reference builds a branch earlier than it consumes it
    assert sorted(a["layers"]) == sorted(b["layers"])
    # and the graph carries the reference-produced weights by name
    G.weight_map(fx, ours)


def test_reference_default_arguments_are_the_same():
    """every keyword and default of the five reference builders exists here with the same default."""
    import inspect
    from deepctr_b200 import models as M
    ref = _golden()["defaults"]
    assert sorted(ref) == sorted(BUILDERS)
    for name in BUILDERS:
        mine = inspect.signature(getattr(M, name))
        assert [k for k, _ in ref[name]] == list(mine.parameters), name
        for k, d in ref[name]:
            assert d == repr(mine.parameters[k].default), (name, k)
