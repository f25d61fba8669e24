#!/usr/bin/env python
"""Generate tests/golden/reference_builders.json: what the reference's five builders build, recorded once so that
tests/test_reference_builders_dropin.py needs no copy of the reference.

    python tests/golden/generate_builders.py /path/to/reference/deepctr

The SOURCE FILES of the builders (deepctr/models/{deepfm,xdeepfm,dcn,autoint}.py, deepctr/models/sequence/din.py)
are executed unmodified with their imports aliased to this package:

    ..feature_column / ..inputs / ..layers.*      ->  deepctr_b200.feature_column / inputs / layers.*
    tensorflow.keras.models.Model, .layers.{Dense,Flatten,Concatenate}  ->  deepctr_b200.engine

For every model fixture the file records the graph they build (inputs, layers, weights, planner slots) and, for
every builder, its keywords with the repr() of their defaults.
"""
import importlib.util
import inspect
import json
import os
import sys
import types

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))

import golden_models as G  # noqa: E402
from golden_models import signature, builder_args  # noqa: E402

_FILES = {"DeepFM": ("models/deepfm.py", "models.deepfm"), "xDeepFM": ("models/xdeepfm.py", "models.xdeepfm"),
          "DCN": ("models/dcn.py", "models.dcn"), "AutoInt": ("models/autoint.py", "models.autoint"),
          "DIN": ("models/sequence/din.py", "models.sequence.din")}


class _aliased(object):
    """sys.modules entries that make the reference builder files import this package; restored on exit."""

    def __enter__(self):
        from deepctr_b200 import engine, feature_column, inputs, layers
        from deepctr_b200.layers import core, interaction, sequence, utils
        self.saved = {k: v for k, v in sys.modules.items() if k == "tensorflow" or k.startswith("tensorflow.")
                      or k == "refdrop" or k.startswith("refdrop.")}
        for k in self.saved:
            del sys.modules[k]

        def mod(name, **attrs):
            m = types.ModuleType(name)
            m.__dict__.update(attrs)
            m.__path__ = []
            sys.modules[name] = m
            return m
        tf = mod("tensorflow")
        tf.keras = mod("tensorflow.keras")
        tf.keras.models = mod("tensorflow.keras.models", Model=engine.Model)
        tf.keras.layers = mod("tensorflow.keras.layers", Dense=engine.Dense, Flatten=engine.Flatten,
                              Concatenate=engine.Concatenate)
        mod("refdrop")
        mod("refdrop.models")
        mod("refdrop.models.sequence")
        sys.modules["refdrop.feature_column"] = feature_column
        sys.modules["refdrop.inputs"] = inputs
        sys.modules["refdrop.layers"] = layers
        sys.modules["refdrop.layers.core"] = core
        sys.modules["refdrop.layers.interaction"] = interaction
        sys.modules["refdrop.layers.sequence"] = sequence
        sys.modules["refdrop.layers.utils"] = utils
        self.added = [k for k in sys.modules if k == "tensorflow" or k.startswith("tensorflow.")
                      or k == "refdrop" or k.startswith("refdrop.")]
        return self

    def __exit__(self, *a):
        for k in self.added:
            sys.modules.pop(k, None)
        sys.modules.update(self.saved)


def _reference_builder(ref, name):
    rel, modname = _FILES[name]
    full = "refdrop." + modname
    spec = importlib.util.spec_from_file_location(full, os.path.join(ref, rel))
    m = importlib.util.module_from_spec(spec)
    sys.modules[full] = m
    spec.loader.exec_module(m)            # the reference's unmodified source
    return getattr(m, name)


def main(ref):
    from deepctr_b200 import engine as E
    out = {"signatures": {}, "defaults": {}}
    with _aliased():
        for name in G.CASES:
            fx = G.Fixture(name)
            args, kw = builder_args(fx)
            build = _reference_builder(ref, fx.builder)
            E.clear_session()
            model = build(*args, **kw)
            G.weight_map(fx, model)          # the reference-built graph carries the fixture's weights by name
            out["signatures"][name] = signature(model)
        for name in G.FAMILIES["models"].builders:
            sig = inspect.signature(_reference_builder(ref, name))
            out["defaults"][name] = [[k, repr(p.default)] for k, p in sig.parameters.items()]
    E.clear_session()
    with open(os.path.join(HERE, "reference_builders.json"), "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)


if __name__ == "__main__":
    main(sys.argv[1])
