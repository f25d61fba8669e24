#!/usr/bin/env python
"""CCPM at the bench shape: 26 single-valued fields x 1M ids, E = 32, no dense features, the reference's defaults
(conv_kernel_width (6, 5), conv_filters (4, 4), DNN (128, 64)), SGD with the fused row-wise update, uniform ids,
batch 65536.

    python tools/ccpm_bench.py [--steps 20] [--warmup 5] [--reps 30]

Prints one JSON line per measurement:
  * the hardware context (card, power limit, max SM clock), read in the same run;
  * b2ctr_conv_stack_fwd / _bwd over the whole default stack, the median over --reps launches, against the two
    bounds counted from the shapes: the bytes they must move at 3.35 TB/s and their FMAs at 67 TFLOP/s FP32
    (H100 SXM data sheet; the backward recomputes the forward);
  * the CCPM training step (graph-replayed once warm) and a DeepFM step at the same shape, for context: device
    time from CUDA events and samples/s.
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import bench  # noqa: E402
from harness import HBM_BYTES_PER_S as HBM, hardware, kernel_ms, time_train_steps  # noqa: E402

FFMA = 67e12
CFG = dict(bench.CONFIGS["c2"], dim=32, n_dense=0,
           workload="CCPM synthetic Criteo: 26 fields x 1M ids, E=32, batch=65536, no dense, reference defaults")
STACK = [("conv", 6, 4, "tanh"), ("kmax", 13), ("conv", 5, 4, "tanh"), ("kmax", 3)]


def _counts(rows):
    """(forward FMAs per column, backward FMAs per column) of STACK on ``rows`` rows: each conv output element
    costs width * C_in FMAs (padding included); the backward recomputes the forward, then dx and the weight gradient
    cost as much again each."""
    fwd, r, c = 0, rows, 1
    for st in STACK:
        if st[0] == "conv":
            fwd += r * st[2] * st[1] * c
            c = st[2]
        else:
            r = st[1]
    return fwd, 3 * fwd


def kernels(reps):
    import torch
    from deepctr_b200 import kernels as K
    B, F, E = CFG["batch"], CFG["n_sparse"], CFG["dim"]
    dev = torch.device("cuda", 0)
    g = torch.Generator(device=dev).manual_seed(0)
    stages, c = [], 1
    for st in STACK:
        if st[0] == "conv":
            stages.append(st + (torch.randn((st[1], 1, c, st[2]), generator=g, device=dev) * 0.3,
                                torch.randn((st[2],), generator=g, device=dev) * 0.1))
            c = st[2]
        else:
            stages.append(st)
    ld = F * E + 4                                   # the embeddings as a window of a wider (gather) buffer
    x = torch.randn((B, ld), generator=g, device=dev)[:, :F * E]
    w_out = 3 * E * 4
    y = torch.empty((B, w_out), device=dev)
    dy = torch.randn((B, w_out), generator=g, device=dev)
    dx = torch.zeros((B, ld), device=dev)[:, :F * E]
    fma_f, fma_b = _counts(F)
    out = []
    for name, fn, nbytes, fma in (
            ("conv_stack_fwd", lambda: K.conv_stack_fwd(stages, x, F, E, 1, B, y), B * 4 * (F * E + w_out),
             fma_f * B * E),
            ("conv_stack_bwd", lambda: K.conv_stack_bwd(stages, x, F, E, 1, B, dy, dx=dx, dx_accumulate=True,
                                                        want_dw=[True, False, True, False]),
             B * 4 * (F * E + w_out + 2 * F * E), fma_b * B * E)):
        ms = float(np.median(kernel_ms(fn, reps)))
        hb, fb = nbytes / HBM * 1e3, 2 * fma / FFMA * 1e3
        out.append({"what": "kernel", "kernel": name, "batch": B, "fields": F, "dim": E, "ms": ms, "bytes": nbytes,
                    "fma": fma, "hbm_bound_ms": hb, "ffma_bound_ms": fb, "x_bound": ms / max(hb, fb)})
    del x, y, dy, dx
    torch.cuda.empty_cache()
    return out


def step(builder, steps, warmup):
    import torch
    from deepctr_b200 import engine as E, models as M
    from deepctr_b200.engine import SGD
    cols = bench.feature_columns(CFG)
    E.clear_session()
    model = getattr(M, builder)(cols, cols, l2_reg_linear=0, l2_reg_embedding=0)
    bench.seed_initializers(model)
    model.compile(SGD(bench.LR), "binary_crossentropy", embedding_update="sparse")
    ms, replayed, _ = time_train_steps(model, CFG, steps, warmup)
    del model
    torch.cuda.empty_cache()
    return {"what": "train_step", "model": builder, "workload": CFG["workload"], "batch": CFG["batch"],
            "steps": steps, "graph_replayed": replayed, "ms_per_step": ms, "samples_per_s": CFG["batch"] / ms * 1e3}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--reps", type=int, default=30)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("ccpm_bench.py measures on an H100: no CUDA device")
    print(json.dumps(dict(what="hardware", **hardware())), flush=True)
    for r in kernels(a.reps):
        print(json.dumps(r), flush=True)
    for b in ("CCPM", "DeepFM"):
        print(json.dumps(step(b, a.steps, a.warmup)), flush=True)


if __name__ == "__main__":
    main()
