#!/usr/bin/env python
"""BST on the C4 synthetic set (bench.py's c4 columns: 100k items, behaviour seq_len 50, emb_dim 64, batch 8192,
history_feature_list=['item_id'], 8 heads of 8), DIN's C4 step for context, and the Transformer kernels at that
shape.

    python tools/bst_bench.py [--steps 20] [--warmup 5] [--reps 50]

Prints one JSON line per measurement:
  * the hardware context (card, power limit, max SM clock), read in the same run;
  * the training step (graph-replayed once warm) of BST and of DIN: device time from CUDA events and samples/s;
  * forward and backward of b2ctr_mha_* and b2ctr_layernorm_*: median over --reps launches, with the HBM bound
    (3.35 TB/s, H100 SXM data sheet) of the bytes the shapes imply and, for the attention, the FFMA bound
    (132 SMs x 128 FP32 lanes x 2 flop x max SM clock) of its flops.
Fails when there is no GPU.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import bench  # noqa: E402
from pairwise_bench import hardware, median_us, HBM_BYTES_PER_S  # noqa: E402


def step_time(builder, steps, warmup):
    import torch
    from deepctr_b200 import engine as E, models as M
    from deepctr_b200.engine import SGD
    cfg = dict(bench.CONFIGS["c4"])
    E.clear_session()
    if builder == "BST":
        model = M.BST(bench.feature_columns(cfg), ["item_id"], att_head_num=8, dnn_hidden_units=cfg["hidden"],
                      l2_reg_embedding=0, l2_reg_dnn=0)
    else:
        model = bench.build_model(cfg)
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
        model.train_step(*batches[(i + k) % bench.N_BATCHES])
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / steps
    res = {"what": "train_step", "model": builder, "batch": cfg["batch"], "steps": steps,
           "graph_replayed": bool(model._step_graphs), "ms_per_step": ms, "samples_per_s": cfg["batch"] / ms * 1e3}
    del model, batches
    torch.cuda.empty_cache()
    return res


def kernels(reps, hw):
    import numpy as np
    import torch
    from deepctr_b200 import kernels as K
    B, T, E, H = 8192, 50, 64, 8
    d = E // H
    dev = torch.device("cuda", 0)
    g = torch.Generator(device=dev).manual_seed(1)
    q, k, v, dout = (torch.randn((B * T, E), device=dev, generator=g) for _ in range(4))
    ln = torch.randint(1, T + 1, (B,), device=dev, generator=g, dtype=torch.int32)
    scale = float(1.0 / np.sqrt(d))
    kw = dict(qlen=ln, klen=ln)
    out, stats = K.mha_fwd(q, E, k, E, v, E, B, T, H, d, scale, res=q, ldr=E, **kw)
    gamma, beta = torch.ones(E, device=dev), torch.zeros(E, device=dev)
    y, lstats = K.layernorm_fwd(out, E, dout, E, gamma, beta, B * T, E, 1e-9)
    clk = hw.get("max_sm_clock_mhz") or None
    ffma_peak = 132 * 128 * 2 * clk * 1e6 if clk else None
    act = B * T * E * 4
    st = B * H * T * 2 * 4
    cases = [
        # Q K^T and P V: 2 * 2 T^2 d per (sample, head); reads Q, K, V and the residual, writes O and the statistics
        ("mha_fwd", lambda: K.mha_fwd(q, E, k, E, v, E, B, T, H, d, scale, res=q, ldr=E, **kw),
         B * H * 4 * T * T * d, 4 * act + act + st),
        # reads Q, K, V, dO and the statistics, writes dQ, dK, dV
        ("mha_bwd", lambda: K.mha_bwd(dout, E, q, E, k, E, v, E, stats, B, T, H, d, scale, **kw),
         None, 4 * act + st + 3 * act),
        # two summands in, y and (mean, rstd) out
        ("layernorm_fwd", lambda: K.layernorm_fwd(out, E, dout, E, gamma, beta, B * T, E, 1e-9),
         None, 3 * act + B * T * 8),
        # two summands, dy and the statistics in, dx out
        ("layernorm_bwd", lambda: K.layernorm_bwd(out, E, dout, E, gamma, lstats, dout, B * T, E),
         None, 4 * act + B * T * 8),
    ]
    res = []
    for name, fn, flops, nbytes in cases:
        med, lo, hi = median_us(fn, reps)
        r = {"what": "kernel", "kernel": name, "shape": "B=%d T=%d E=%d heads=%d" % (B, T, E, H),
             "median_us": med, "min_us": lo, "max_us": hi, "bytes": nbytes,
             "hbm_bound_us": nbytes / HBM_BYTES_PER_S * 1e6}
        if flops is not None:
            r["flops"] = flops
            r["ffma_bound_us"] = flops / ffma_peak * 1e6 if ffma_peak else None
        bound = max(r["hbm_bound_us"], r.get("ffma_bound_us") or 0.0)
        r["share_of_bound"] = bound / med
        res.append(r)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--reps", type=int, default=50)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bst_bench: no CUDA device; nothing here can be measured without an H100")
    torch.cuda.set_device(0)
    hw = hardware()
    print(json.dumps(dict(what="hardware", **hw)), flush=True)
    for builder in ("BST", "DIN"):
        print(json.dumps(step_time(builder, a.steps, a.warmup)), flush=True)
    for r in kernels(a.reps, hw):
        print(json.dumps(r), flush=True)


if __name__ == "__main__":
    main()
