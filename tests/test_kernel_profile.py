"""CPU: the per-kernel profile (kernels.PROFILE, bench.py's kernel_ms_per_step) takes each call of a wrapper that
enqueues device work as one entry under the wrapper's name.  No kernels are launched: the C library is a fake."""
import inspect

import torch

from deepctr_b200 import _lib as L, kernels as K

# a synchronising read of the out-of-range id counter, not a launch to attribute
UNTIMED = {"embed_oob_count"}


def _calls_the_c_abi(fn):
    src = inspect.getsource(getattr(fn, "__wrapped__", fn))
    return "_lib_call(" in src or "L.lib().b2ctr_" in src


def test_every_launching_wrapper_is_timed_once():
    public = {n: f for n, f in vars(K).items()
              if inspect.isfunction(f) and not n.startswith("_") and f.__module__ == K.__name__}
    launching = {n for n, f in public.items() if _calls_the_c_abi(f)}
    assert {"gemm", "ewise", "cin_gemm", "fm_weighted_fwd", "pack_rows", "embed_oob_count"} <= launching
    untimed = sorted(n for n in launching - UNTIMED if not hasattr(public[n], "__wrapped__"))
    twice = sorted(n for n in launching - UNTIMED if hasattr(getattr(public[n], "__wrapped__", None), "__wrapped__"))
    assert not untimed, "launching wrappers without @_timed: %s" % untimed
    assert not twice, "wrappers timed twice: %s" % twice
    assert not hasattr(K.embed_oob_count, "__wrapped__")


class _FakeLib(object):
    def __getattr__(self, name):
        return lambda *args: L.OK


class _FakeEvent(object):
    def __init__(self, enable_timing=False):
        pass

    def record(self):
        pass


def test_each_call_records_one_entry(monkeypatch):
    monkeypatch.setattr(L, "_lib", _FakeLib())
    monkeypatch.setattr(torch.cuda, "Event", _FakeEvent)
    monkeypatch.setattr(K, "stream", lambda: None)
    monkeypatch.setattr(K, "_require_cuda", lambda *tensors: None)
    B, F, E = 4, 3, 2
    x, m = torch.zeros((B, F * E)), torch.ones((B, F))
    with K.profiled() as prof:
        K.ewise(0, x, x)
        K.bi_interaction_fwd(x, F * E, F, E, B)
        K.fm_weighted_fwd(x, F * E, m, F, E, B)
        with K.profile_tag("cin"):
            K.cin_sum_d(x, F * E, 0, F * E, E, x, F * E, 0, 0, B)
    assert K.PROFILE is None
    assert {k: len(v) for k, v in prof.items()} == {"ewise": 1, "bi_interaction_fwd": 1, "fm_weighted_fwd": 1,
                                                    "cin:cin_sum_d": 1}
