#!/usr/bin/env python
"""NFM / AFM / FiBiNET on the C2 synthetic set (26 tables x 1M rows, emb_dim 32, batch 65536, uniform ids; NFM and
FiBiNET also get the 13 dense features, AFM takes none: its builder refuses DenseFeat) and the pairwise kernels at
that shape.

    python tools/pairwise_bench.py [--steps 20] [--warmup 5] [--reps 50] [--models NFM,AFM,FiBiNET]
    python tools/pairwise_bench.py --models FwFM,DeepFEFM
    python tools/pairwise_bench.py --models PNN
    python tools/pairwise_bench.py --models IFM,DIFM

Prints one JSON line per measurement:
  * the hardware context (card, power limit, max SM clock), read in the same run;
  * the training step (graph-replayed once warm) of NFM (256, 128, 64) and AFM (attention_factor 8): device time
    from CUDA events and samples/s;
  * forward and backward of b2ctr_afm_*, b2ctr_bi_interaction_*, b2ctr_senet_* and b2ctr_bilinear_* (each type):
    median over --reps launches, with the FFMA bound (132 SMs x 128 FP32 lanes x 2 flop x max SM clock) and the HBM
    bound (3.35 TB/s, H100 SXM data sheet) of the flops and bytes their shapes imply;
  * FiBiNET's first DNN layer alone: the split of its [65536, 20816] operand into bf16 planes and the three
    20813 -> 256 GEMMs (forward, data gradient, weight gradient), so the step can be broken down;
  * with FwFM / DeepFEFM (not in the default set): b2ctr_fwfm_* and b2ctr_fefm_* against the same two bounds, and the
    training steps of FwFM and DeepFEFM with their default (256, 128, 64) DNN;
  * with PNN (not in the default set): b2ctr_pnn_inner_* (inner, vec, num) and b2ctr_pnn_outer_* (mat) against the
    same two bounds, and the training steps of IPNN (the default), OPNN with kernel_type 'mat' and both products,
    with the (256, 128, 64) DNN;
  * with IFM / DIFM (not in the default set): b2ctr_fm_weighted_*, b2ctr_field_scale_* (E = 32 and the linear term's
    E = 1) and b2ctr_softmax_rows_* against the HBM bound, and the training steps of IFM and DIFM (13 dense features,
    (256, 128, 64) DNN).
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402
from harness import HBM_BYTES_PER_S, hardware, kernel_ms, time_train_steps  # noqa: E402

# --models PNN: the three product configurations timed
PNN_STEPS = {"PNN-inner": dict(use_inner=True, use_outter=False),
             "PNN-outer-mat": dict(use_inner=False, use_outter=True, kernel_type="mat"),
             "PNN-inner-outer-mat": dict(use_inner=True, use_outter=True, kernel_type="mat")}


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
    elif builder == "FwFM":
        model = M.FwFM(cols, cols, dnn_hidden_units=(256, 128, 64), l2_reg_linear=0, l2_reg_embedding=0)
    elif builder == "DeepFEFM":
        model = M.DeepFEFM(cols, cols, dnn_hidden_units=(256, 128, 64), l2_reg_linear=0, l2_reg_embedding_feat=0)
    elif builder.startswith("PNN"):
        model = M.PNN(cols, dnn_hidden_units=(256, 128, 64), l2_reg_embedding=0, **PNN_STEPS[builder])
    elif builder in ("IFM", "DIFM"):
        model = getattr(M, builder)(cols, cols, dnn_hidden_units=(256, 128, 64), l2_reg_linear=0, l2_reg_embedding=0)
    elif builder == "FiBiNET":
        model = M.FiBiNET(cols, cols, bilinear_type="interaction", dnn_hidden_units=(256, 128, 64), l2_reg_linear=0,
                          l2_reg_embedding=0)
    else:
        model = M.AFM(cols, cols, attention_factor=8, l2_reg_linear=0, l2_reg_embedding=0, l2_reg_att=0)
    bench.seed_initializers(model)
    model.compile(SGD(bench.LR), "binary_crossentropy", embedding_update="sparse")
    ms, replayed, loss = time_train_steps(model, cfg, steps, warmup)
    del model
    torch.cuda.empty_cache()
    return {"what": "train_step", "model": builder, "batch": cfg["batch"], "steps": steps, "graph_replayed": replayed,
            "ms_per_step": ms, "samples_per_s": cfg["batch"] / ms * 1e3, "loss": loss}


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
    shape = dict(B=B, F=F, E=E, A=A, ldx=ld)
    return [_report(name, shape, reps, fn, flops, nbytes, ffma_peak) for name, fn, flops, nbytes in cases]


def _report(name, shape, reps, fn, flops, nbytes, ffma_peak):
    ts = np.array(kernel_ms(fn, reps)) * 1e3
    return {"what": "kernel", "kernel": name, "shape": shape, "reps": reps, "median_us": float(np.median(ts)),
            "min_us": float(ts.min()), "max_us": float(ts.max()), "flops": flops, "bytes": nbytes,
            "hbm_bound_us": nbytes / HBM_BYTES_PER_S * 1e6,
            "ffma_bound_us": flops / ffma_peak * 1e6 if ffma_peak else None}


def fibinet_kernels(reps, hw):
    """SENET and the bilinear kernels at C2 (26 fields, E = 32, B = 65536), the pairs written into the [B, 20816]
    DNN input as FiBiNET places them; then the split and the GEMMs of the 20813 -> 256 first layer."""
    import torch
    from deepctr_b200 import _lib as L, kernels as K, ops
    B, F, E, nd, R = 65536, 26, 32, 13, 8
    P = F * (F - 1) // 2
    dev = torch.device("cuda", 0)
    g = torch.Generator(device=dev).manual_seed(2)
    clk = hw.get("max_sm_clock_mhz") or None
    ffma_peak = 132 * 128 * 2 * clk * 1e6 if clk else None
    ldx = F * E + nd + 3
    buf = torch.randn((B, ldx), device=dev, generator=g) * 0.1
    xw = buf[:, :F * E]
    W1 = torch.randn((F, R), device=dev, generator=g) * 0.3
    W2 = torch.randn((R, F), device=dev, generator=g) * 0.3
    kd = 2 * P * E + nd
    ld = (kd + 3) // 4 * 4
    dnn_in = torch.randn((B, ld), device=dev, generator=g) * 0.1       # also the bilinear outputs' gradient
    shape = dict(B=B, F=F, E=E, P=P, ldx=ldx, ld_out=ld)
    x_bytes, v_bytes = B * F * E * 4, B * F * E * 4
    v, saved = K.senet_fwd(xw, ldx, F, E, W1, W2, B)
    out = [_report("senet_fwd", shape, reps, lambda: K.senet_fwd(xw, ldx, F, E, W1, W2, B),
                   B * (F * E * 2 + 4 * F * R), x_bytes + v_bytes + B * (R + F) * 4, ffma_peak),
           _report("senet_bwd", shape, reps, lambda: K.senet_bwd(v, xw, ldx, F, E, W1, W2, saved, B),
                   B * (F * E * 6 + 8 * F * R), 3 * x_bytes + B * (R + F) * 4, ffma_peak)]
    pair_bytes = B * P * E * 4
    for t in ("all", "each", "interaction"):
        nw = 1 if t == "all" else F - 1 if t == "each" else P
        W = torch.randn((nw, E, E), device=dev, generator=g) / E ** 0.5
        # forward: (v_i W) per pair 2E^2 + the product E; backward: dx (2 x 2E^2 + E), dW (2E^2 + E) per pair
        out.append(_report("bilinear_fwd_" + t, shape, reps,
                           lambda: K.bilinear_fwd(xw, ldx, F, E, t, W, B, out=dnn_in, col0=0, pitch=2 * E),
                           B * P * (2 * E * E + E), x_bytes + pair_bytes, ffma_peak))
        gv = dnn_in[:, E:]
        out.append(_report("bilinear_bwd_" + t, shape, reps,
                           lambda: K.bilinear_bwd(gv, ld, 0, 2 * E, xw, ldx, F, E, t, W, B),
                           B * P * (6 * E * E + 3 * E), 2 * x_bytes + 3 * pair_bytes, ffma_peak))
        del W
    # the first DNN layer 20813 -> 256 on the placed buffer, timed alone
    n = 256
    x2 = dnn_in[:, :kd]
    w = torch.randn((kd, n), device=dev, generator=g) / kd ** 0.5
    dz = torch.randn((B, n), device=dev, generator=g) / B
    xp, wp, dzp = K.split_planes(x2), K.split_planes(w), K.split_planes(dz)
    gshape = dict(m=B, k=kd, n=n, ld=ld)
    bf = L.GEMM_BF16X3
    dxbuf = torch.empty((B, ld), device=dev)
    gemm_flops = 2 * B * kd * n
    out.append(_report("split_planes_dnn_input", gshape, reps, lambda: K.split_planes(x2), 0,
                       B * kd * 4 + B * kd * 4, ffma_peak))
    out.append(_report("gemm_fwd_20813x256", gshape, reps,
                       lambda: K.gemm(x2, w, act=L.ACT_RELU, precision=bf, m=B, n=n, k=kd, a_planes=xp, b_planes=wp),
                       gemm_flops, B * kd * 4 + B * n * 4, None))
    out.append(_report("gemm_dgrad_20813x256", gshape, reps,
                       lambda: K.gemm(dz, w, c=dxbuf[:, :kd], trans_b=True, precision=bf, m=B, n=kd, k=n,
                                      a_planes=dzp, b_planes=wp),
                       gemm_flops, B * kd * 4 + B * n * 4, None))
    out.append(_report("gemm_wgrad_20813x256", gshape, reps,
                       lambda: K.gemm(x2, dz, trans_a=True, precision=bf, split_k=ops._split_k(kd, n, B), m=kd, n=n,
                                      k=B, a_planes=xp, b_planes=dzp),
                       gemm_flops, B * kd * 4 + B * n * 4, None))
    del buf, dnn_in, xp, dxbuf
    torch.cuda.empty_cache()
    return out


def fefm_kernels(reps, hw):
    """FwFM and FEFM at C2 (26 fields, E = 32, B = 65536), x a window of the [B, 848] gather buffer and FEFM's scores
    written at column 845 of a [B, 1172] buffer, as DeepFEFM's DNN input holds them."""
    import torch
    from deepctr_b200 import kernels as K
    B, F, E, nd = 65536, 26, 32, 13
    P = F * (F - 1) // 2
    dev = torch.device("cuda", 0)
    g = torch.Generator(device=dev).manual_seed(3)
    clk = hw.get("max_sm_clock_mhz") or None
    ffma_peak = 132 * 128 * 2 * clk * 1e6 if clk else None
    ldx = (F * E + nd + 3) // 4 * 4
    buf = torch.randn((B, ldx), device=dev, generator=g) * 0.1
    xw = buf[:, :F * E]
    x_bytes = B * F * E * 4
    shape = dict(B=B, F=F, E=E, P=P, ldx=ldx)
    r = torch.randn((F, F), device=dev, generator=g) * 0.3
    gl = torch.randn((B, 1), device=dev, generator=g)
    # FwFM: 2E flop per pair; the backward recomputes the dots for dR (2E per pair) and forms dx (2E per pair, twice)
    out = [_report("fwfm_fwd", shape, reps, lambda: K.fwfm_fwd(xw, ldx, F, E, r, B), B * P * 2 * E,
                   x_bytes + B * 4, ffma_peak),
           _report("fwfm_bwd", shape, reps, lambda: K.fwfm_bwd(gl, 1, xw, ldx, F, E, r, B), B * P * 6 * E,
                   2 * x_bytes + B * 4, ffma_peak)]
    W = torch.randn((P, E, E), device=dev, generator=g) / E ** 0.5
    S = K.fefm_sym(W)
    ld, col0 = (F * E + nd + P + 3) // 4 * 4, F * E + nd
    dnn_in = torch.randn((B, ld), device=dev, generator=g) * 0.1       # also the scores' gradient
    shape = dict(shape, ld_out=ld, col0=col0)
    w_bytes = P * E * E * 4
    out.append(_report("fefm_sym", dict(P=P, E=E), reps, lambda: K.fefm_sym(W), P * E * E, 3 * w_bytes, ffma_peak))
    # forward: x_i S_p 2E^2 + the dot 2E per pair; backward: dx 2 x (2E^2 + E), dS 2E^2 + E per pair
    out.append(_report("fefm_fwd", shape, reps, lambda: K.fefm_fwd(xw, ldx, F, E, S, B, out=dnn_in, col0=col0),
                       B * P * (2 * E * E + 2 * E), x_bytes + w_bytes + B * P * 4, ffma_peak))
    out.append(_report("fefm_bwd", shape, reps, lambda: K.fefm_bwd(dnn_in, ld, col0, xw, ldx, F, E, S, B),
                       B * P * (6 * E * E + 3 * E), 2 * x_bytes + 2 * w_bytes + B * P * 4, ffma_peak))
    del buf, dnn_in, W, S
    torch.cuda.empty_cache()
    return out


def pnn_kernels(reps, hw):
    """PNN's products at C2 (26 fields, E = 32, B = 65536), x a window of the [B, 848] gather buffer and the scores
    written at column 845 of a [B, 1172] buffer."""
    import torch
    from deepctr_b200 import kernels as K
    B, F, E, nd = 65536, 26, 32, 13
    P = F * (F - 1) // 2
    dev = torch.device("cuda", 0)
    g = torch.Generator(device=dev).manual_seed(4)
    clk = hw.get("max_sm_clock_mhz") or None
    ffma_peak = 132 * 128 * 2 * clk * 1e6 if clk else None
    ldx = (F * E + nd + 3) // 4 * 4
    buf = torch.randn((B, ldx), device=dev, generator=g) * 0.1
    xw = buf[:, :F * E]
    x_bytes, s_bytes = B * F * E * 4, B * P * 4
    ld, col0 = (F * E + nd + P + 3) // 4 * 4, F * E + nd
    dnn_in = torch.randn((B, ld), device=dev, generator=g) * 0.1       # also the scores' gradient
    shape = dict(B=B, F=F, E=E, P=P, ldx=ldx, ld_out=ld, col0=col0)
    out = []
    # inner / vec / num: 2E flop per pair forward; backward dx 2E per pair and field (twice), dK 2E (vec) per pair
    for mode, Kw in (("inner", None), ("vec", torch.randn((P, E), device=dev, generator=g) / E ** 0.5),
                     ("num", torch.randn((P, 1), device=dev, generator=g))):
        k_bytes = 0 if Kw is None else Kw.numel() * 4
        out.append(_report("pnn_inner_fwd_" + mode, shape, reps,
                           lambda: K.pnn_inner_fwd(xw, ldx, F, E, mode, Kw, B, out=dnn_in, col0=col0),
                           B * P * 2 * E, x_bytes + s_bytes + k_bytes, ffma_peak))
        out.append(_report("pnn_inner_bwd_" + mode, shape, reps,
                           lambda: K.pnn_inner_bwd(dnn_in, ld, col0, xw, ldx, F, E, mode, Kw, B),
                           B * P * (4 * E + (2 * E if Kw is not None else 0)), 2 * x_bytes + s_bytes + 2 * k_bytes,
                           ffma_peak))
    Km = torch.randn((E, P, E), device=dev, generator=g) / E ** 0.5
    k_bytes = Km.numel() * 4
    # mat, the FEFM tiles: forward x_i M_p 2E^2 + the dot 2E per pair; backward dx 2 x (2E^2 + E), dK 2E^2 + E
    out.append(_report("pnn_outer_fwd_mat", shape, reps,
                       lambda: K.pnn_outer_fwd(xw, ldx, F, E, Km, B, out=dnn_in, col0=col0),
                       B * P * (2 * E * E + 2 * E), x_bytes + k_bytes + s_bytes, ffma_peak))
    out.append(_report("pnn_outer_bwd_mat", shape, reps,
                       lambda: K.pnn_outer_bwd(dnn_in, ld, col0, xw, ldx, F, E, Km, B),
                       B * P * (6 * E * E + 3 * E), 2 * x_bytes + 2 * k_bytes + s_bytes, ffma_peak))
    del buf, dnn_in, Km
    torch.cuda.empty_cache()
    return out


def ifm_kernels(reps, hw):
    """IFM / DIFM's field-weight kernels at C2 (26 fields, E = 32, B = 65536), x a window of the [B, 848] gather
    buffer: the field-weighted FM (backward with and without accumulate into the buffer's gradient), the
    materialised field scale at E = 32 (what the deferred FM avoids) and at E = 1 (the linear term), and IFM's
    F * softmax over [B, 26]."""
    import torch
    from deepctr_b200 import kernels as K
    B, F, E, nd = 65536, 26, 32, 13
    dev = torch.device("cuda", 0)
    g = torch.Generator(device=dev).manual_seed(5)
    clk = hw.get("max_sm_clock_mhz") or None
    ffma_peak = 132 * 128 * 2 * clk * 1e6 if clk else None
    ldx = (F * E + nd + 3) // 4 * 4
    buf = torch.randn((B, ldx), device=dev, generator=g) * 0.1
    dbuf = torch.randn((B, ldx), device=dev, generator=g)
    xw, dxw = buf[:, :F * E], dbuf[:, :F * E]
    m = torch.randn((B, F), device=dev, generator=g)
    go = torch.randn((B,), device=dev, generator=g)
    x_bytes, m_bytes = B * F * E * 4, B * F * 4
    shape = dict(B=B, F=F, E=E, ldx=ldx)
    out = [_report("fm_weighted_fwd", shape, reps, lambda: K.fm_weighted_fwd(xw, ldx, m, F, E, B),
                   B * F * E * 4, x_bytes + m_bytes + B * 4, ffma_peak),
           _report("fm_weighted_bwd", shape, reps, lambda: K.fm_weighted_bwd(xw, ldx, m, F, E, go, B, dx=dxw),
                   B * F * E * 8, 2 * x_bytes + 2 * m_bytes + B * 4, ffma_peak),
           _report("fm_weighted_bwd_accumulate", shape, reps,
                   lambda: K.fm_weighted_bwd(xw, ldx, m, F, E, go, B, dx=dxw, accumulate=True),
                   B * F * E * 8, 3 * x_bytes + 2 * m_bytes + B * 4, ffma_peak)]
    y = K.field_scale_fwd(xw, ldx, m, F, E, B)
    out += [_report("field_scale_fwd", shape, reps, lambda: K.field_scale_fwd(xw, ldx, m, F, E, B, out=y),
                    B * F * E, 2 * x_bytes + m_bytes, ffma_peak),
            _report("field_scale_bwd", shape, reps, lambda: K.field_scale_bwd(y, xw, ldx, m, F, E, B, dx=dxw),
                    B * F * E * 3, 3 * x_bytes + 2 * m_bytes, ffma_peak)]
    lin = torch.randn((B, 28), device=dev, generator=g)
    shape1 = dict(B=B, F=F, E=1, ldx=28)
    out += [_report("field_scale_fwd_e1", shape1, reps, lambda: K.field_scale_fwd(lin, 28, m, F, 1, B),
                    B * F, 3 * m_bytes, ffma_peak),
            _report("field_scale_bwd_e1", shape1, reps, lambda: K.field_scale_bwd(m, lin, 28, m, F, 1, B),
                    B * F * 3, 5 * m_bytes, ffma_peak)]
    sm = K.softmax_rows_fwd(m, float(F))
    shape_s = dict(B=B, C=F)
    out += [_report("softmax_rows_fwd", shape_s, reps, lambda: K.softmax_rows_fwd(m, float(F)), B * F * 5,
                    2 * m_bytes, ffma_peak),
            _report("softmax_rows_bwd", shape_s, reps, lambda: K.softmax_rows_bwd(sm, m, float(F)), B * F * 4,
                    3 * m_bytes, ffma_peak)]
    del buf, dbuf, y
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--models", default="NFM,AFM,FiBiNET")
    args = ap.parse_args()
    models = args.models.split(",")
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("pairwise_bench.py needs a CUDA device")
    hw = hardware()
    print(json.dumps(dict(what="hardware", **hw)), flush=True)
    if "NFM" in models or "AFM" in models:
        for r in kernels(args.reps, hw):
            print(json.dumps(r), flush=True)
    if "FiBiNET" in models:
        for r in fibinet_kernels(args.reps, hw):
            print(json.dumps(r), flush=True)
    if "FwFM" in models or "DeepFEFM" in models:
        for r in fefm_kernels(args.reps, hw):
            print(json.dumps(r), flush=True)
    if "PNN" in models:
        for r in pnn_kernels(args.reps, hw):
            print(json.dumps(r), flush=True)
        models = [m for m in models if m != "PNN"] + list(PNN_STEPS)
    if "IFM" in models or "DIFM" in models:
        for r in ifm_kernels(args.reps, hw):
            print(json.dumps(r), flush=True)
    for builder in models:
        print(json.dumps(step_time(builder, args.steps, args.warmup)), flush=True)


if __name__ == "__main__":
    main()
