#!/usr/bin/env python
"""ONN at the bench shape: 26 single-valued fields x 1M ids, E = 4 (650 tables of [1M, 4], 10.4 GB), 13 dense
features, the (256, 128, 64) DNN, use_bn=True, SGD with the fused row-wise update, uniform ids, batch 65536.

    python tools/onn_bench.py [--steps 20] [--warmup 5] [--reps 30]

Prints one JSON line per measurement:
  * the hardware context (card, power limit, max SM clock), read in the same run;
  * b2ctr_ffm_product_fwd (elementwise and reduce_sum) and b2ctr_ffm_product_bwd (elementwise) at that shape, the
    median over --reps launches, against two HBM bounds at 3.35 TB/s (H100 SXM data sheet): the algorithmic one
    (ids, 650 rows of 16 B, the output; the backward also the gradient, 650 partner rows and the 2 x 650 x 16 B of
    the scratch it writes) and the sector one (every 16 B row read costs a 32 B sector);
  * the scatter that applies the backward's scratch (b2ctr_embed_scatter_add, fused SGD), timed the same way;
  * the ONN training step (graph-replayed once warm): device time from CUDA events and samples/s.
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

CFG = dict(bench.CONFIGS["c2"], dim=4, workload="ONN synthetic Criteo: 26 fields x 1M ids, E=4, batch=65536, 13 dense")


def kernels(reps):
    import torch
    from deepctr_b200 import kernels as K
    B, F, E, V = CFG["batch"], CFG["n_sparse"], CFG["dim"], CFG["vocab"]
    P = F * (F - 1) // 2
    dev = torch.device("cuda", 0)
    tables = [None] * (F * F)
    for a in range(F):
        for b in range(F):
            if a != b:
                tables[a * F + b] = torch.randn((V, E), device=dev) * 0.01
    ptrs = torch.tensor([t.data_ptr() if t is not None else 0 for t in tables], dtype=torch.int64, device=dev)
    rng = np.random.RandomState(0)
    ids = [torch.from_numpy(rng.randint(0, V, size=B).astype(np.int32)).to(dev) for _ in range(F)]
    out = []
    row, sector, idb = E * 4, 32, 4
    for reduce_sum in (False, True):
        w = P if reduce_sum else P * E
        o = torch.empty((B, (w + 3) // 4 * 4), device=dev)      # the planner's pitch: a multiple of 4 floats
        fields = [K.ffm_field(idx=i, vocab=V) for i in ids]
        ms = float(np.median(kernel_ms(lambda: K.ffm_product_fwd(fields, ptrs, E, reduce_sum, o, 0, B), reps)))
        alg = B * (F * idb + 2 * P * row + w * 4)
        sec = B * (F * idb + 2 * P * sector + w * 4)
        out.append({"what": "kernel", "kernel": "ffm_product_fwd", "mode": "reduce_sum" if reduce_sum else
                    "elementwise", "batch": B, "fields": F, "dim": E, "ms": ms, "bytes_algorithmic": alg,
                    "hbm_bound_ms": alg / HBM * 1e3, "bytes_sectors": sec, "sector_bound_ms": sec / HBM * 1e3,
                    "x_algorithmic_bound": ms / (alg / HBM * 1e3), "x_sector_bound": ms / (sec / HBM * 1e3)})
    g = torch.randn((B, P * E), device=dev)
    scratch = torch.empty((B, F * (F - 1) * E), device=dev)
    fields = [K.ffm_field(idx=i, vocab=V, grad=scratch[:, a * (F - 1) * E:]) for a, i in enumerate(ids)]
    ms = float(np.median(kernel_ms(lambda: K.ffm_product_bwd(fields, ptrs, E, False, g, 0, B), reps)))
    alg = B * (F * idb + P * E * 4 + 2 * P * row + 2 * P * row)
    sec = B * (F * idb + P * E * 4 + 2 * P * sector + 2 * P * row)
    out.append({"what": "kernel", "kernel": "ffm_product_bwd", "mode": "elementwise", "batch": B, "fields": F,
                "dim": E, "ms": ms, "bytes_algorithmic": alg, "hbm_bound_ms": alg / HBM * 1e3,
                "bytes_sectors": sec, "sector_bound_ms": sec / HBM * 1e3,
                "x_algorithmic_bound": ms / (alg / HBM * 1e3), "x_sector_bound": ms / (sec / HBM * 1e3)})
    feats = []
    for a in range(F):
        for b in range(F):
            if a != b:
                s = b - (b > a)
                feats.append(K.make_feature(tables[a * F + b], ids[a], scratch, out_col=(a * (F - 1) + s) * E,
                                            out_ld=scratch.stride(0), vocab=V))

    ms = float(np.median(kernel_ms(lambda: K.embed_scatter_add(feats, B, -1e-6), reps)))
    # reads the scratch and the ids, read-modify-writes 650 rows (each a 32 B sector) per sample
    alg = B * (2 * P * row + 2 * P * idb + 2 * 2 * P * row)
    out.append({"what": "kernel", "kernel": "embed_scatter_add (ONN scratch, fused SGD)", "batch": B,
                "lookups": F * (F - 1), "ms": ms, "bytes_algorithmic": alg, "hbm_bound_ms": alg / HBM * 1e3,
                "x_algorithmic_bound": ms / (alg / HBM * 1e3)})
    del tables, ptrs, scratch, g
    torch.cuda.empty_cache()
    return out


def step(steps, warmup):
    from deepctr_b200 import engine as E, models as M
    from deepctr_b200.engine import SGD
    cols = bench.feature_columns(CFG)
    E.clear_session()
    model = M.ONN(cols, cols, dnn_hidden_units=(256, 128, 64), l2_reg_linear=0, l2_reg_embedding=0)
    bench.seed_initializers(model)
    model.compile(SGD(bench.LR), "binary_crossentropy", embedding_update="sparse")
    ms, replayed, _ = time_train_steps(model, CFG, steps, warmup)
    return {"what": "train_step", "model": "ONN", "workload": CFG["workload"], "batch": CFG["batch"],
            "steps": steps, "graph_replayed": replayed, "ms_per_step": ms, "samples_per_s": CFG["batch"] / ms * 1e3}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--reps", type=int, default=30)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("onn_bench.py measures on an H100: no CUDA device")
    print(json.dumps(dict(what="hardware", **hardware())), flush=True)
    for r in kernels(a.reps):
        print(json.dumps(r), flush=True)
    print(json.dumps(step(a.steps, a.warmup)), flush=True)


if __name__ == "__main__":
    main()
