#!/usr/bin/env python
"""The fused embedding kernels of the C2 step alone (26 tables x 1M rows, emb_dim 32, 13 dense features, batch 65536,
uniform ids), against the HBM data sheet and against two ceilings measured on the same tables:

    python tools/embed_bench.py [--reps 50] [--batch 65536]

Prints one JSON line per measurement (median of --reps launches, CUDA events):
  * the hardware context (card, power limit, max SM clock), read in the same run;
  * ceilings: ``copy`` = the uniform gather with FM, linear term and dense passthrough off (random 128-byte row reads
    plus the X write), ``red`` = the uniform scatter with only dX (dX read plus one random 128-byte red.add per row);
  * ``gather``: the gather as the C2 step runs it (X, FM, linear term, dense passthrough), ``gather+S+planes`` with
    the FM sum vectors and X's bf16 planes written as well;
  * ``scatter``: the update re-summing S from X, ``scatter+S`` reading the gather's S;
  * ``split_planes``: the split of X [65536, 845] into its bf16 planes, which ``gather+S+planes`` makes unnecessary.
Each line gives the bytes the kernel has to move (32-byte sectors, 64 for the linear term's red), GB/s, and the
fraction of the data sheet (3.35 TB/s, H100 SXM) and of the measured ceiling of its kind (reads and writes: copy,
updates: red).
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from harness import HBM_BYTES_PER_S, hardware, kernel_ms  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--batch", type=int, default=65536)
    a = ap.parse_args()
    import torch
    from deepctr_b200 import kernels as K, _lib as L
    torch.cuda.set_device(0)
    dev = torch.device("cuda", 0)
    F, V, E, ND, B = 26, 1 << 20, 32, 13, a.batch
    kd = F * E + ND
    ldx = (kd + 3) // 4 * 4
    g = torch.Generator(device=dev).manual_seed(0)
    tabs = [torch.randn((V, E), device=dev, generator=g) * 0.01 for _ in range(F)]
    lins = [torch.randn((V,), device=dev, generator=g) * 0.01 for _ in range(F)]
    ids = torch.randint(0, V, (B, F), device=dev, generator=g, dtype=torch.int32)
    dense = torch.rand((B, ND), device=dev, generator=g)
    x = torch.empty((B, ldx), device=dev)
    fm, linear = torch.empty((B,), device=dev), torch.empty((B,), device=dev)
    dx = torch.randn((B, ldx), device=dev, generator=g) * 1e-3
    dfm, dlin = torch.randn((B,), device=dev, generator=g) * 1e-3, torch.randn((B,), device=dev, generator=g) * 1e-3
    feats = [K.make_feature(tabs[f], ids[:, f], x, out_col=f * E, out_ld=ldx, vocab=V) for f in range(F)]
    full = (1 << F) - 1

    def plan(lin=True, dn=True, with_fm=True):
        p = K.UniformPlan(feats, lins if lin else None, dense if dn else None, x, linear if lin else None,
                          fm if with_fm else None, full if with_fm else 0)
        p.g.x_cols = ldx
        return p

    # bytes per sample: 32-byte sectors; the linear term touches one 64-byte granule per lookup
    row, ids_b, xrow = E * 4, F * 4, ldx * 4
    lin_rd, lin_rmw = F * 64, 2 * F * 64
    planes_row = L.lib().b2ctr_planes_bytes(B, kd) // ((B + 255) // 256 * 256)     # hi + lo, padded pitch
    traffic = {
        "copy": ids_b + F * row + xrow,
        "red": ids_b + F * E * 4 + 2 * F * row,
        "gather": ids_b + F * row + lin_rd + ND * 4 + xrow + 8,
        "gather+S+planes": ids_b + F * row + lin_rd + ND * 4 + xrow + 8 + E * 4 + planes_row,
        "scatter": ids_b + 2 * F * E * 4 + 2 * F * row + lin_rmw + 8,
        "scatter+S": ids_b + 2 * F * E * 4 + 2 * F * row + lin_rmw + 8 + E * 4,
        "split_planes": kd * 4 + planes_row,
    }

    p_copy = plan(lin=False, dn=False, with_fm=False)
    p_gather = plan()
    p_gather.fm_sum = None
    p_full = plan()
    have_ex = hasattr(p_full, "set_planes")
    if have_ex:
        p_full.set_planes(kd)
    K.embed_gather_uniform_fwd(p_full, B)
    # the updates land in scratch copies so the tables stay as the gathers read them
    gt = [torch.zeros_like(t) for t in tabs]
    glin = [torch.zeros_like(t) for t in lins]
    bfeats = [K.make_feature(gt[f], ids[:, f], x, out_col=f * E, out_ld=ldx, vocab=V) for f in range(F)]
    b_red = K.UniformPlan(bfeats, None, None, x, None, None, full)
    b_full = K.UniformPlan(bfeats, glin, None, x, None, None, full)
    x2 = x[:, :kd]
    runs = {
        "copy": lambda: K.embed_gather_uniform_fwd(p_copy, B),
        "red": lambda: K.embed_scatter_uniform_bwd(b_red, dx, None, None, -1e-3, -1e-3, B),
        "gather": lambda: K.embed_gather_uniform_fwd(p_gather, B),
        "scatter": lambda: K.embed_scatter_uniform_bwd(b_full, dx, dfm, dlin, -1e-3, -1e-3, B),
        "split_planes": lambda: K.split_planes(x2),
    }
    if have_ex:
        runs["gather+S+planes"] = lambda: K.embed_gather_uniform_fwd(p_full, B)
        runs["scatter+S"] = lambda: K.embed_scatter_uniform_bwd(b_full, dx, dfm, dlin, -1e-3, -1e-3, B,
                                                                fm_sum=p_full.fm_sum)
    print(json.dumps(dict(hardware(), shape=dict(F=F, V=V, E=E, ndense=ND, batch=B), tree=ROOT)), flush=True)
    us = {k: float(np.median(kernel_ms(fn, a.reps))) * 1e3 for k, fn in runs.items()}
    ceil = {k: traffic[k] * B / (us[k] * 1e-6) for k in ("copy", "red")}
    for k, t in us.items():
        nbytes = traffic[k] * B
        rate = nbytes / (t * 1e-6)
        kind = "red" if k.startswith("scatter") or k == "red" else "copy"
        print(json.dumps({"kernel": k, "us": round(t, 1), "MB": round(nbytes / 1e6, 1), "GB_s": round(rate / 1e9, 1),
                          "frac_datasheet": round(rate / HBM_BYTES_PER_S, 3),
                          "frac_ceiling_" + kind: round(rate / ceil[kind], 3)}), flush=True)


if __name__ == "__main__":
    main()
