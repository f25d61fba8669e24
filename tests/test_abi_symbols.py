"""CPU: the C-ABI library loads and exports every symbol include/b2ctr.h declares, and the ctypes
struct mirrors have the sizes the header documents.  No compute calls (no GPU here)."""
import ctypes
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared():
    src = open(os.path.join(ROOT, "include", "b2ctr.h")).read()
    return sorted(set(re.findall(r"B2CTR_API\s+[\w\s\*]+?\b(b2ctr_\w+)\s*\(", src)))


def test_abi_v2_symbols_are_exported_and_bound():
    from deepctr_b200 import _lib as L
    names = _declared()
    assert len(names) >= 20
    handle = L.lib()  # raises if the .so is missing: there is no fallback
    for n in names:
        assert hasattr(handle, n), "libb2ctr.so does not export %s" % n
        assert n in L.SIGNATURES, "_lib.SIGNATURES lacks %s" % n
    assert set(L.SIGNATURES) == set(names)
    assert handle.b2ctr_abi_version() == 2
    assert handle.b2ctr_last_error() is not None


def test_abi_v2_struct_layouts_match_header():
    from deepctr_b200 import _lib as L
    assert ctypes.sizeof(L.Feature) == 112
    assert L.Feature.src_table.offset == 96
    assert ctypes.sizeof(L.Gemm) == 128
    assert ctypes.sizeof(L.UniformGather) == 120


def test_kernels_refuse_cpu_tensors():
    import pytest
    import torch
    from deepctr_b200 import kernels as K, _lib as L
    with pytest.raises(L.B2ctrError):
        K.act_fwd(torch.zeros(4), L.ACT_RELU)
