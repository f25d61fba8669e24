#!/usr/bin/env python
"""EDCN at the bench shape: 26 single-valued fields x 1M ids, E = 16 (d = 416), no dense features (EDCN rejects
them), cross_num = 2, SGD with the fused row-wise update, uniform ids, batch 65536, for each bridge type.

    python tools/edcn_bench.py [--steps 20] [--warmup 5] [--reps 30]

Prints one JSON line per measurement:
  * the hardware context (card, power limit, max SM clock), read in the same run;
  * b2ctr_regulate_fwd / _bwd in the launches the planner issues: 'copy' with both gates (layer 0's pair on the
    gather buffer, dx added to its gradient) and each bridge mode with both gates (an inner boundary), the median
    over --reps launches against the HBM bound of the bytes they must move at 3.35 TB/s (H100 SXM data sheet);
  * the EDCN training step per bridge type (graph-replayed once warm): device time from CUDA events and samples/s.
"""
import argparse
import contextlib
import functools
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import bench  # noqa: E402
from harness import HBM_BYTES_PER_S as HBM, hardware, kernel_ms, time_train_steps  # noqa: E402

CFG = dict(bench.CONFIGS["c2"], dim=16, n_dense=0,
           workload="EDCN synthetic Criteo: 26 fields x 1M ids, E=16, batch=65536, no dense, cross_num=2")
BRIDGES = ("pointwise_addition", "hadamard_product", "concatenation", "attention_pooling")
# operands each mode reads
N_IN = {"copy": 1, "add": 2, "hadamard": 2, "attention": 4}


def kernels(reps):
    import torch
    from deepctr_b200 import kernels as K
    B, F, E = CFG["batch"], CFG["n_sparse"], CFG["dim"]
    d = F * E
    dev = torch.device("cuda", 0)
    ops_ = [torch.rand((B, d), device=dev) for _ in range(4)]
    gates = [(torch.randn((F,), device=dev), 1.0) for _ in range(2)]
    y0, y1, dy0, dy1 = (torch.randn((B, d), device=dev) for _ in range(4))
    dx = torch.zeros((B, d), device=dev)
    out = []
    for mode, n_in in N_IN.items():
        x, h, ax, ah = [ops_[k] if k < n_in else None for k in range(4)]
        fwd = functools.partial(K.regulate_fwd, mode, F, E, B, x, h, ax, ah, gates, y0=(y0, 0), y1=(y1, 0))
        ms = float(np.median(kernel_ms(fwd, reps)))
        nbytes = B * d * 4 * (n_in + 2)
        out.append({"what": "kernel", "kernel": "regulate_fwd", "mode": mode, "outputs": "y0,y1", "batch": B,
                    "fields": F, "dim": E, "ms": ms, "bytes": nbytes, "hbm_bound_ms": nbytes / HBM * 1e3,
                    "x_hbm_bound": ms / (nbytes / HBM * 1e3)})
        acc = mode == "copy"             # layer 0 adds dx to the gather buffer's gradient
        bwd = functools.partial(K.regulate_bwd, mode, F, E, B, x, h, ax, ah, gates, dy0=(dy0, 0), dy1=(dy1, 0),
                                dx=dx if acc else None, dx_accumulate=acc, want_dh=h is not None,
                                want_dax=ax is not None, want_dah=ah is not None, want_dg=(True, True))
        ms = float(np.median(kernel_ms(bwd, reps)))
        nbytes = B * d * 4 * (n_in + 2 + n_in + (1 if acc else 0))
        out.append({"what": "kernel", "kernel": "regulate_bwd", "mode": mode, "outputs": "y0,y1", "batch": B,
                    "fields": F, "dim": E, "ms": ms, "bytes": nbytes, "hbm_bound_ms": nbytes / HBM * 1e3,
                    "x_hbm_bound": ms / (nbytes / HBM * 1e3)})
    del ops_, y0, y1, dy0, dy1, dx
    torch.cuda.empty_cache()
    return out


def step(bridge_type, steps, warmup):
    import torch
    from deepctr_b200 import engine as E, models as M
    from deepctr_b200.engine import SGD
    cols = bench.feature_columns(CFG)
    E.clear_session()
    with contextlib.redirect_stdout(sys.stderr):          # the builder's prints stay off the JSON lines
        model = M.EDCN(cols, cols, cross_num=2, bridge_type=bridge_type, l2_reg_linear=0, l2_reg_embedding=0)
    bench.seed_initializers(model)
    model.compile(SGD(bench.LR), "binary_crossentropy", embedding_update="sparse")
    ms, replayed, _ = time_train_steps(model, CFG, steps, warmup)
    del model
    torch.cuda.empty_cache()
    return {"what": "train_step", "model": "EDCN", "bridge_type": bridge_type, "workload": CFG["workload"],
            "batch": CFG["batch"], "steps": steps, "graph_replayed": replayed, "ms_per_step": ms,
            "samples_per_s": CFG["batch"] / ms * 1e3}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--reps", type=int, default=30)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("edcn_bench.py measures on an H100: no CUDA device")
    print(json.dumps(dict(what="hardware", **hardware())), flush=True)
    for r in kernels(a.reps):
        print(json.dumps(r), flush=True)
    for bt in BRIDGES:
        print(json.dumps(step(bt, a.steps, a.warmup)), flush=True)


if __name__ == "__main__":
    main()
