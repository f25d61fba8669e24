#!/usr/bin/env python
"""The DNN tower after its first layer at C2's shape: (256, 128, 64) relu layers, batch 65536.

    python tools/tower_bench.py [--reps 30] [--parent DIR]

Prints one JSON line per measurement:
  * the hardware context (card, power limit, max SM clock), read in the same run;
  * the eager launch list of one C2 training step (harness.launch_list): launches and CUDA-event ms per kernel
    wrapper; with --parent, also the launch list of the checkout at DIR (another commit of this repository, built);
  * b2ctr_mlp_relu_fwd and b2ctr_mlp_relu_bwd, the median over --reps launches, against their HBM floors at
    3.35 TB/s (H100 SXM data sheet) counted from the shapes:
      forward:  read y0 fp32; write the planes of y0 and y1 (hi + lo bf16) and y2 fp32;
      backward: read dy2 and y2 fp32, y1's hi plane (its relu mask) and y0 fp32 (its mask); write the planes of
                dz2, dz1 and dz0.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TOOLS = os.path.join(ROOT, "tools")


def _setup(root):
    sys.path.insert(0, TOOLS)
    sys.path.insert(0, root)


def launches():
    import torch
    import bench
    from harness import launch_list
    from deepctr_b200 import engine as E
    from deepctr_b200.engine import SGD
    cfg = bench.CONFIGS["c2"]
    E.clear_session()
    model = bench.build_model(cfg)
    bench.seed_initializers(model)
    model.compile(SGD(bench.LR), "binary_crossentropy", embedding_update="sparse")
    x, y = next(iter(bench.synth_batches(cfg, 1)))
    lst = launch_list(model, bench.device_inputs(cfg, x, y, torch.device("cuda", 0)))
    return {"what": "launch_list", "config": "c2", "tree": os.path.abspath(sys.path[0]), "launches": lst,
            "total_launches": sum(v["launches"] for v in lst.values()),
            "total_ms": round(sum(v["ms"] for v in lst.values()), 4)}


def kernels(reps):
    import numpy as np
    import torch
    from harness import HBM_BYTES_PER_S as HBM, kernel_ms
    from deepctr_b200 import kernels as K
    B, (n0, n1, n2) = 65536, (256, 128, 64)
    dev = torch.device("cuda", 0)
    g = torch.Generator(device=dev)
    g.manual_seed(0)
    y0 = torch.relu(torch.randn((B, n0), generator=g, device=dev))
    ws = [torch.randn((n0, n1), generator=g, device=dev) * n0 ** -0.5,
          torch.randn((n1, n2), generator=g, device=dev) * n1 ** -0.5]
    bs = [torch.randn((n1,), generator=g, device=dev) * 0.1, torch.randn((n2,), generator=g, device=dev) * 0.1]
    dy = torch.randn((B, n2), generator=g, device=dev)
    planes, y = K.mlp_relu_fwd(y0, ws, bs)
    fwd_bytes = B * (n0 * 4 + n0 * 4 + n1 * 4 + n2 * 4)
    bwd_bytes = B * (n2 * 4 + n2 * 4 + n1 * 2 + n0 * 4 + (n0 + n1 + n2) * 4)
    flop = 2 * 3 * B * (n0 * n1 + n1 * n2)
    out = []
    for name, fn, nbytes in (("mlp_relu_fwd", lambda: K.mlp_relu_fwd(y0, ws, bs), fwd_bytes),
                             ("mlp_relu_bwd", lambda: K.mlp_relu_bwd(dy, y, y0, planes, ws), bwd_bytes)):
        ms = float(np.median(kernel_ms(fn, reps)))
        out.append({"what": "kernel", "kernel": name, "batch": B, "widths": [n0, n1, n2], "ms": ms,
                    "bytes": nbytes, "hbm_floor_ms": nbytes / HBM * 1e3, "x_floor": ms / (nbytes / HBM * 1e3),
                    "bf16_mma_flop": flop})
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--parent", default=None, help="another built checkout whose C2 launch list to print too")
    ap.add_argument("--launches-only", default=None, help=argparse.SUPPRESS)   # child run for --parent
    a = ap.parse_args()
    if a.launches_only:
        _setup(a.launches_only)
        print(json.dumps(launches()), flush=True)
        return
    _setup(ROOT)
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("tower_bench.py measures on an H100: no CUDA device")
    from harness import hardware
    print(json.dumps(dict(what="hardware", **hardware())), flush=True)
    if a.parent:
        subprocess.run([sys.executable, os.path.abspath(__file__), "--launches-only", os.path.abspath(a.parent)],
                       check=True)
    print(json.dumps(launches()), flush=True)
    for r in kernels(a.reps):
        print(json.dumps(r), flush=True)


if __name__ == "__main__":
    main()
