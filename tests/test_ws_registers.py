"""CPU: the plain persistent split-bf16 GEMM kernels keep everything in registers.

Their ping-pong consumer warpgroups hold two m64nBN accumulators (128 registers per thread at BN = 128) and take
the registers the producer warpgroup gives up (setmaxnreg).  If the budgets stop fitting, ptxas spills to local
memory, which no numerical test sees; this reads the resource usage of the built library instead."""
import os
import re
import subprocess

import pytest

from test_sass_pipeline import LIB, WS, _cuobjdump


def test_plain_ws_kernels_use_no_stack():
    exe = _cuobjdump()
    if exe is None:
        pytest.skip("cuobjdump not found")
    if not os.path.exists(LIB):
        pytest.skip("libb2ctr.so not built")
    out = subprocess.run([exe, "-res-usage", LIB], check=True, capture_output=True, text=True).stdout
    plain, name = {}, None
    for line in out.splitlines():
        m = re.search(r"Function (\S+):", line)
        if m:
            name = m.group(1)
            continue
        k = WS.search(name or "")
        if k and k.group(3) == "0" and k.group(4) == "0":
            res = dict(re.findall(r"(\w+(?:\[\d+\])?):(\d+)", line))
            if res:
                plain[name] = res
                name = None
    assert sorted(int(WS.search(n).group(1)) for n in plain) == [32, 64, 128], sorted(plain)
    bad = {n: (r["STACK"], r["LOCAL"]) for n, r in plain.items() if r["STACK"] != "0" or r["LOCAL"] != "0"}
    assert not bad, bad
