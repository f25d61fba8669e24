"""CPU: the fused relu-tower kernels keep their A fragments and accumulators in registers.

Each warp holds a whole layer's output as the next product's A operand; if that stops fitting, ptxas spills to local
memory, which no numerical test sees.  This reads the resource usage of the built library instead."""
import os
import re
import subprocess

import pytest

from test_sass_pipeline import LIB, _cuobjdump

TOWER = re.compile(r"mlp_relu_(fwd|bwd)_kernelILi(\d+)ELi(\d+)ELi(\d+)E")


def test_tower_kernels_use_no_stack():
    exe = _cuobjdump()
    if exe is None:
        pytest.skip("cuobjdump not found")
    if not os.path.exists(LIB):
        pytest.skip("libb2ctr.so not built")
    out = subprocess.run([exe, "-res-usage", LIB], check=True, capture_output=True, text=True).stdout
    found, name = {}, None
    for line in out.splitlines():
        m = re.search(r"Function (\S+):", line)
        if m:
            name = m.group(1)
            continue
        if name and TOWER.search(name):
            res = dict(re.findall(r"(\w+(?:\[\d+\])?):(\d+)", line))
            if res:
                found[TOWER.search(name).groups()] = res
                name = None
    towers = {(int(a), int(b), int(c)) for _, a, b, c in found}
    assert {(256, 128, 64)} <= towers and len(found) == 2 * len(towers), sorted(found)
    bad = {k: (r["STACK"], r["LOCAL"]) for k, r in found.items() if r["STACK"] != "0" or r["LOCAL"] != "0"}
    assert not bad, bad
