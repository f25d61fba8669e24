"""Per-shape timing of the split-bf16 wgmma GEMM (CUDA events, caller-provided planes as ops.dense passes
them) for the C2 DeepFM layer shapes: forward / dgrad / wgrad of 845->256->128->64 at batch 65536.
usage: python tools/gemm_bench.py [variants...]   (default: 3 4; 3 = non-persistent reference, 4 = persistent)"""
import sys

import torch
sys.path.insert(0, ".")
from deepctr_b200 import _lib as L, kernels as K

B = 65536
LAYERS = [(845, 256), (256, 128), (128, 64)]


def shapes():
    out = []
    for kin, nout in LAYERS:
        out.append(("fwd  %4d->%-4d" % (kin, nout), B, nout, kin, False, False, 1))
        out.append(("dgrad%4d->%-4d" % (kin, nout), B, kin, nout, False, True, 1))
        tiles = ((kin + 255) // 256) * ((nout + 255) // 256)
        out.append(("wgrad%4d->%-4d" % (kin, nout), kin, nout, B, True, False, max(1, min(74 // tiles, B // 1024))))
    return out


def main():
    variants = [int(v) for v in sys.argv[1:]] or [3, 4]
    dev = torch.device("cuda")
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    print("%-18s %8s %8s" % ("shape", "m,n,k", "") + "".join("   v%d us (TF/s bf16-eq)" % v for v in variants))
    import os
    only = os.environ.get("GEMM_BENCH_ONLY")
    for idx, (name, m, n, k, ta, tb, sk) in enumerate(shapes()):
        if only is not None and idx != int(only):
            continue
        a = torch.randn((k, m) if ta else (m, k), device=dev)
        b = torch.randn((n, k) if tb else (k, n), device=dev)
        ap, bp = K.split_planes(a), K.split_planes(b)
        cbuf = torch.empty((m, (n + 7) // 8 * 8), device=dev)      # 16-byte aligned rows, as the model's buffers
        cview = cbuf[:, :n]
        row = "%-18s %6d %5d %6d sk=%-3d" % (name, m, n, k, sk)
        for v in variants:
            def run():
                return K.gemm(a, b, c=cview, trans_a=ta, trans_b=tb, precision=L.GEMM_BF16X3, m=m, n=n, k=k,
                              split_k=sk, variant=v, a_planes=ap, b_planes=bp)
            for _ in range(3):
                run()
            ts = []
            for _ in range(10):
                flush.zero_()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                run()
                e1.record()
                torch.cuda.synchronize()
                ts.append(e0.elapsed_time(e1) * 1e3)
            ts.sort()
            us = ts[len(ts) // 2]
            row += "   %8.1f (%6.0f)" % (us, 3 * 2.0 * m * n * k / us / 1e6)
        print(row)


if __name__ == "__main__":
    main()
