#!/usr/bin/env python
"""NFM / AFM on the C2 synthetic set (26 tables x 1M rows, emb_dim 32, batch 65536, uniform ids; NFM also gets the
13 dense features, AFM takes none: its builder refuses DenseFeat) and the fused pairwise kernels at that shape.

    python tools/pairwise_bench.py [--steps 20] [--warmup 5] [--reps 50]

Prints one JSON line per measurement:
  * the hardware context (card, power limit, max SM clock), read in the same run;
  * the training step (graph-replayed once warm) of NFM (256, 128, 64) and AFM (attention_factor 8): device time
    from CUDA events and samples/s;
  * forward and backward of b2ctr_afm_* and b2ctr_bi_interaction_*: median over --reps launches, with the FFMA bound
    (132 SMs x 128 FP32 lanes x 2 flop x max SM clock) and the HBM bound (3.35 TB/s, H100 SXM data sheet) of the
    flops and bytes their shapes imply.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402

HBM_BYTES_PER_S = 3.35e12


def hardware():
    import torch
    out = {"card": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader,nounits",
                            "-i", "0"], capture_output=True, text=True, timeout=30).stdout.strip().split(",")
        out["power_limit_w"] = float(q[0])
        out["max_sm_clock_mhz"] = float(q[1])
    except Exception as e:      # the numbers are then reported as unknown, never guessed
        out["power_limit_w"] = out["max_sm_clock_mhz"] = None
        out["query_error"] = repr(e)
    return out


def step_time(builder, steps, warmup):
    import torch
    from deepctr_b200 import engine as E, models as M
    from deepctr_b200.engine import SGD
    cfg = dict(bench.CONFIGS["c2"])
    if builder == "AFM":
        cfg["n_dense"] = 0
    cols = bench.feature_columns(cfg)
    E.clear_session()
    if builder == "NFM":
        model = M.NFM(cols, cols, dnn_hidden_units=(256, 128, 64), l2_reg_linear=0, l2_reg_embedding=0)
    else:
        model = M.AFM(cols, cols, attention_factor=8, l2_reg_linear=0, l2_reg_embedding=0, l2_reg_att=0)
    bench.seed_initializers(model)
    model.compile(SGD(bench.LR), "binary_crossentropy", embedding_update="sparse")
    dev = torch.device("cuda", 0)
    batches = [bench.device_inputs(cfg, x, y, dev) for x, y in bench.synth_batches(cfg, bench.N_BATCHES)]
    i = 0
    while i < warmup or (i < warmup + bench.N_BATCHES + 4 and model._graph_eligible()
                         and len(model._step_graphs) < bench.N_BATCHES):
        model.train_step(*batches[i % bench.N_BATCHES])
        i += 1
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for k in range(steps):
        loss = model.train_step(*batches[(i + k) % bench.N_BATCHES])
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / steps
    res = {"what": "train_step", "model": builder, "batch": cfg["batch"], "steps": steps,
           "graph_replayed": bool(model._step_graphs), "ms_per_step": ms,
           "samples_per_s": cfg["batch"] / ms * 1e3, "loss": float(loss[0]) if isinstance(loss, tuple) else None}
    del model, batches
    torch.cuda.empty_cache()
    return res


def median_us(fn, reps):
    import torch
    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b) * 1e3)
    return float(np.median(ts)), float(np.min(ts)), float(np.max(ts))


def kernels(reps, hw):
    import torch
    from deepctr_b200 import kernels as K
    B, F, E, A, nd = 65536, 26, 32, 8, 13
    P = F * (F - 1) // 2
    dev = torch.device("cuda", 0)
    g = torch.Generator(device=dev).manual_seed(1)
    ld = F * E + nd + 3                      # the gather buffer: [B, F*E | 13 dense | pad]
    buf = torch.randn((B, ld), device=dev, generator=g) * 0.1
    xw = buf[:, :F * E]
    W = torch.randn((E, A), device=dev, generator=g) / E ** 0.5
    b = torch.zeros(A, device=dev)
    h = torch.randn(A, device=dev, generator=g)
    gatt = torch.randn((B, E), device=dev, generator=g) / B
    att, state = K.afm_fwd(xw, ld, F, E, W, b, h, B)
    clk = hw.get("max_sm_clock_mhz") or None
    ffma_peak = 132 * 128 * 2 * clk * 1e6 if clk else None
    x_bytes = F * E * 4
    cases = [
        # per pair: product E, scores 2EA + 2A, online softmax + weighted sum 2E
        ("afm_fwd", lambda: K.afm_fwd(xw, ld, F, E, W, b, h, B),
         B * P * (E + 2 * E * A + 2 * A + 2 * E), B * (x_bytes + E * 4 + 8)),
        # per pair: product E, scores 2EA + 2A, <g, prod> 2E, d prod 2EA + E, dW 2EA, dx fold 4E, ~6A
        ("afm_bwd", lambda: K.afm_bwd(gatt, xw, ld, F, E, W, b, h, state, att, B),
         B * P * (6 * E * A + 8 * E + 8 * A), B * (2 * x_bytes + 2 * E * 4 + 8)),
        ("bi_interaction_fwd", lambda: K.bi_interaction_fwd(xw, ld, F, E, B),
         B * F * E * 3, B * (x_bytes + E * 4)),
        ("bi_interaction_bwd", lambda: K.bi_interaction_bwd(xw, ld, F, E, gatt, B),
         B * F * E * 3, B * (2 * x_bytes + E * 4)),
    ]
    out = []
    for name, fn, flops, nbytes in cases:
        med, lo, hi = median_us(fn, reps)
        r = {"what": "kernel", "kernel": name, "shape": dict(B=B, F=F, E=E, A=A, ldx=ld), "reps": reps,
             "median_us": med, "min_us": lo, "max_us": hi, "flops": flops, "bytes": nbytes,
             "hbm_bound_us": nbytes / HBM_BYTES_PER_S * 1e6,
             "ffma_bound_us": flops / ffma_peak * 1e6 if ffma_peak else None}
        out.append(r)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--reps", type=int, default=50)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("pairwise_bench.py needs a CUDA device")
    hw = hardware()
    print(json.dumps(dict(what="hardware", **hw)), flush=True)
    for r in kernels(args.reps, hw):
        print(json.dumps(r), flush=True)
    for builder in ("NFM", "AFM"):
        print(json.dumps(step_time(builder, args.steps, args.warmup)), flush=True)


if __name__ == "__main__":
    main()
