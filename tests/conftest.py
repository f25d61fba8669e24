import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (ROOT, os.path.join(ROOT, 'tests')):
    if _p not in sys.path:
        sys.path.insert(0, _p)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (run with -m gpu)")


@pytest.fixture(scope="session")
def cuda():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda:0")


# Model-level GPU parity runs in BOTH GEMM precisions: 'bf16x3' (the default: wgmma split-bf16, what bench.py
# measures) and 'fp32' (exact FFMA path).  Modules opt in with:  from conftest import gemm_precision  # noqa
@pytest.fixture(params=["bf16x3", "fp32"], autouse=False)
def gemm_precision(request):
    from deepctr_b200 import ops
    ops.set_gemm_precision(request.param)
    yield request.param
    ops.set_gemm_precision("bf16x3")
