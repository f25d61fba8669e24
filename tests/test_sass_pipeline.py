"""CPU: the split-bf16 wgmma kernels keep one k-block's MMAs in flight while the next one is issued.

Each 64-deep k-block issues 12 wgmma (4 K-steps x hi*hi, hi*lo, lo*hi) and commits them as one group; the
persistent kernel then waits for all but the newest group (wgmma.wait_group 1), so consecutive k-blocks overlap on
the tensor pipe.  If the compiler cannot prove the accumulator registers untouched between the MMAs and their
commit (a control-flow join, an accumulator access), it closes the group early and commits an empty one
(`HGMMA.64x8x16.F16 RZ`), and the wait then retires the k-block just issued.  No numerical test can see that, so
this reads the SASS of the built library."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "deepctr_b200", "libb2ctr.so")
KTK_MMAS = 12          # wgmma per k-block: 64 / 16 K-steps x 3 products
# gemm_planes_ws_kernel<BN, STAGES, GEN, FOLD>
WS = re.compile(r"gemm_planes_ws_kernelILi(\d+)ELi(\d+)ELi(\d+)ELb([01])E")


def _cuobjdump():
    exe = shutil.which("cuobjdump")
    if exe is None and os.path.exists("/usr/local/cuda/bin/cuobjdump"):
        exe = "/usr/local/cuda/bin/cuobjdump"
    return exe


@pytest.fixture(scope="module")
def sass():
    exe = _cuobjdump()
    if exe is None:
        pytest.skip("cuobjdump not found")
    if not os.path.exists(LIB):
        pytest.skip("libb2ctr.so not built")
    out = subprocess.run([exe, "-sass", LIB], check=True, capture_output=True, text=True).stdout
    funcs, name = {}, None
    for line in out.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            name = m.group(1)
            funcs[name] = []
        elif name is not None:
            m = re.search(r"/\*[0-9a-f]{4,}\*/\s+(.*?)\s*;", line)
            if m:
                funcs[name].append(m.group(1))
    return funcs


def _kernels(funcs, stem):
    return {k: v for k, v in funcs.items() if stem in k}


def _groups(instrs):
    """(number of HGMMAs, number of group-closing HGMMAs, number of empty groups, waits after each group)"""
    n_mma = n_close = n_empty = 0
    waits = []
    for i, ins in enumerate(instrs):
        if not ins.startswith("HGMMA"):
            continue
        if " RZ, gdesc[URZ]" in ins:
            n_empty += 1
            continue
        n_mma += 1
        if ins.endswith("gsb0"):
            n_close += 1
            # the first warpgroup-sync instruction after the group's commit
            nxt = next((s for s in instrs[i + 1:] if s.startswith(("HGMMA", "WARPGROUP"))), None)
            waits.append(nxt)
    return n_mma, n_close, n_empty, waits


def test_ws_kernels_overlap_consecutive_kblocks(sass):
    ws = _kernels(sass, "gemm_planes_ws_kernel")
    # (BN, GEN, FOLD): plain BN 32 / 64 / 128, CIN (GEN 1) and attention (GEN 2) BN 64 / 128, and the CIN fold
    got = sorted((int(WS.search(n).group(1)), int(WS.search(n).group(3)), WS.search(n).group(4) == "1") for n in ws)
    assert got == sorted([(32, 0, False), (64, 0, False), (128, 0, False), (64, 1, False), (128, 1, False),
                          (64, 2, False), (128, 2, False), (128, 0, True)]), sorted(ws)
    for name, instrs in ws.items():
        n_mma, n_close, n_empty, waits = _groups(instrs)
        assert n_empty == 0, "%s: %d empty wgmma groups" % (name, n_empty)
        assert n_close > 0 and n_mma == KTK_MMAS * n_close, (name, n_mma, n_close)
        # after committing k-block kb, wait for kb - 1 only
        bad = [w for w in waits if w != "WARPGROUP.DEPBAR.LE gsb0, 0x1"]
        assert not bad, "%s: a k-block's group is followed by %s" % (name, bad[0])


@pytest.mark.parametrize("stem", ["gemm_planes_kernel"])
def test_other_wgmma_kernels_commit_one_group_per_kblock(sass, stem):
    ks = _kernels(sass, stem)
    assert ks, stem
    for name, instrs in ks.items():
        n_mma, n_close, n_empty, _ = _groups(instrs)
        assert n_empty == 0, "%s: %d empty wgmma groups" % (name, n_empty)
        assert n_close > 0 and n_mma == KTK_MMAS * n_close, (name, n_mma, n_close)
