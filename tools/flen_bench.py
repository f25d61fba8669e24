#!/usr/bin/env python
"""FLEN at the bench shapes, SGD with the fused row-wise update, uniform ids, batch 65536:
  * c2_interleaved: 26 fields x 1M ids, E = 32, 13 dense, groups i % 3 (the reference tests' grouping);
  * c2_contiguous:  the same fields in three contiguous groups (9, 9, 8); the difference between the two is what
    combined_dnn_input's group-major concatenation costs when the groups interleave in the gather buffer;
  * run_flen:       examples/run_flen.py's 21 fields in its three groups, E = 16, 1M ids, no dense.

    python tools/flen_bench.py [--steps 20] [--warmup 5] [--reps 30]

Prints one JSON line per measurement:
  * the hardware context (card, power limit, max SM clock), read in the same run;
  * b2ctr_field_wise_bi_fwd / _bwd at the C2 shape, the median over --reps launches, against the bytes they must
    move at 3.35 TB/s (H100 SXM data sheet): the forward reads x and writes h, the backward reads x and dh and
    read-modify-writes dx in the [B, 848] gather buffer's gradient;
  * the FLEN training step per shape (graph-replayed once warm): device time from CUDA events and samples/s;
  * the launch list of one eager training step at the interleaved C2 shape.
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
from harness import HBM_BYTES_PER_S as HBM, hardware, kernel_ms, launch_list, time_train_steps  # noqa: E402

C2 = dict(bench.CONFIGS["c2"], dim=32)
RUN_FLEN_GROUPS = ("context", "user", "context", "context", "context", "context", "item", "item", "item", "user",
                   "user", "user", "context", "user", "user", "user", "user", "user", "user", "user", "user")
SHAPES = {
    "c2_interleaved": (dict(C2, workload="FLEN synthetic Criteo: 26 fields x 1M ids, E=32, 13 dense, groups i % 3"),
                       [str(i % 3) for i in range(26)]),
    "c2_contiguous": (dict(C2, workload="FLEN synthetic Criteo: 26 fields x 1M ids, E=32, 13 dense, 3 contiguous "
                                        "groups"), [str(i * 3 // 26) for i in range(26)]),
    "run_flen": (dict(C2, n_sparse=21, n_dense=0, dim=16,
                      workload="FLEN run_flen.py layout: 21 fields x 1M ids in 3 groups, E=16, no dense"),
                 list(RUN_FLEN_GROUPS)),
}


def kernels(reps):
    import torch
    from deepctr_b200 import kernels as K
    B, F, E = C2["batch"], C2["n_sparse"], C2["dim"]
    ld = 848                                          # the gather buffer: 26 x 32 embeddings, 13 dense, padding
    dev = torch.device("cuda", 0)
    g = torch.Generator(device=dev).manual_seed(0)
    x = torch.randn((B, ld), generator=g, device=dev)
    cols, groups = [f * E for f in range(F)], [f % 3 for f in range(F)]
    kmf, kfm = torch.ones((3, 1), device=dev), torch.full((3, 1), 0.5, device=dev)
    bmf, bfm = torch.zeros((E,), device=dev), torch.zeros((E,), device=dev)
    h = torch.empty((B, E), device=dev)
    dh = torch.randn((B, E), generator=g, device=dev)
    dx = torch.zeros((B, ld), device=dev)
    out = []
    for name, fn, nbytes in (
            ("field_wise_bi_fwd", lambda: K.field_wise_bi_fwd(x, cols, groups, 3, E, B, kmf, kfm, bmf, bfm, h),
             B * 4 * (F * E + E)),
            ("field_wise_bi_bwd", lambda: K.field_wise_bi_bwd(x, cols, groups, 3, E, B, kmf, kfm, bmf, bfm, dh,
                                                              dx=dx, dx_accumulate=True, want_dkernel=(True, True),
                                                              want_dbias=(True, True)),
             B * 4 * (F * E + E + 2 * F * E))):
        ms = float(np.median(kernel_ms(fn, reps)))
        hb = nbytes / HBM * 1e3
        out.append({"what": "kernel", "kernel": name, "batch": B, "fields": F, "groups": 3, "dim": E, "ms": ms,
                    "bytes": nbytes, "hbm_bound_ms": hb, "x_bound": ms / hb})
    del x, h, dh, dx
    torch.cuda.empty_cache()
    return out


def _model(cfg, groups, step_graph="auto"):
    from deepctr_b200 import engine as E, models as M
    from deepctr_b200.engine import SGD
    cols = bench.feature_columns(cfg)
    cols = [c._replace(group_name=groups[i]) if i < len(groups) else c for i, c in enumerate(cols)]
    E.clear_session()
    model = M.FLEN(cols, cols, l2_reg_linear=0, l2_reg_embedding=0)
    bench.seed_initializers(model)
    model.compile(SGD(bench.LR), "binary_crossentropy", embedding_update="sparse", step_graph=step_graph)
    return model


def step(name, steps, warmup):
    import torch
    cfg, groups = SHAPES[name]
    model = _model(cfg, groups)
    ms, replayed, _ = time_train_steps(model, cfg, steps, warmup)
    del model
    torch.cuda.empty_cache()
    return {"what": "train_step", "model": "FLEN", "shape": name, "workload": cfg["workload"], "batch": cfg["batch"],
            "steps": steps, "graph_replayed": replayed, "ms_per_step": ms, "samples_per_s": cfg["batch"] / ms * 1e3}


def step_launches(name):
    import torch
    cfg, groups = SHAPES[name]
    model = _model(cfg, groups, step_graph="off")
    (x, y), = bench.synth_batches(cfg, 1)
    launches = launch_list(model, bench.device_inputs(cfg, x, y, torch.device("cuda", 0)))
    del model
    torch.cuda.empty_cache()
    return {"what": "launch_list", "shape": name, "step": launches}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--reps", type=int, default=30)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("flen_bench.py measures on an H100: no CUDA device")
    print(json.dumps(dict(what="hardware", **hardware())), flush=True)
    for r in kernels(a.reps):
        print(json.dumps(r), flush=True)
    for name in SHAPES:
        print(json.dumps(step(name, a.steps, a.warmup)), flush=True)
    print(json.dumps(step_launches("c2_interleaved")), flush=True)


if __name__ == "__main__":
    main()
