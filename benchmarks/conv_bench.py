#!/usr/bin/env python
"""Per-layer timing of the implicit-GEMM convolution (csrc/conv_sm90.cu) against cuDNN on the
ResNet-50 shapes at batch 256 (the headline config): forward, dgrad, wgrad.

    python benchmarks/conv_bench.py [--batch 256] [--iters 10] [--out conv_bench.json]

Timing: CUDA events on the launching stream, 3 warm-up calls, an L2 flush (256 MiB memset) before
every timed call.  TFLOP/s = 2*N*OH*OW*Cout*Cin*R*S / t; fraction is against
MEASURED_PEAKS.json ``bf16_tflops`` (burst, since each kernel is timed in isolation).
"""
import argparse
import json
import os
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

SHAPES = [  # Cin, H, W, Cout, R, stride      (ResNet-50 v1.5, 224x224)
    (64, 56, 56, 64, 3, 1),
    (128, 56, 56, 128, 3, 2),
    (128, 28, 28, 128, 3, 1),
    (256, 28, 28, 256, 3, 2),
    (256, 14, 14, 256, 3, 1),
    (512, 14, 14, 512, 3, 2),
    (512, 7, 7, 512, 3, 1),
    (256, 56, 56, 512, 1, 2),
    (512, 28, 28, 1024, 1, 2),
    (1024, 14, 14, 2048, 1, 2),
]


def timeit(fn, iters, flush):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        flush.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    ts.sort()
    return ts[len(ts) // 2] * 1e3   # median, us


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--out", default=None, help="also write the rows to this JSON file")
    ap.add_argument("--only", type=int, default=-1, help="run a single shape index")
    ap.add_argument("--ours-only", action="store_true", help="skip the cuDNN arm (for ncu captures)")
    args = ap.parse_args()
    from distributed_torch_horovod_gcp_b200.ops import kernels, conv as C
    assert kernels.has("conv_implicit_gemm")
    peak = 989.0      # H100 SXM data sheet, dense bf16 (not measured); MEASURED_PEAKS.json overrides
    try:
        peak = json.load(open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))),
                                           "MEASURED_PEAKS.json")))["bf16_tflops"]
    except Exception:
        pass
    torch.backends.cudnn.benchmark = True
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    rows = []
    N = args.batch
    shapes = SHAPES if args.only < 0 else [SHAPES[args.only]]
    for (ci, H, W, co, R, s) in shapes:
        pad = (R - 1) // 2
        x = torch.randn(N, ci, H, W, device="cuda").to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
        w = (torch.randn(co, ci, R, R, device="cuda") * 0.05).to(torch.bfloat16).contiguous(
            memory_format=torch.channels_last)
        y = C.conv_fprop(x, w, s, pad)
        dy = torch.randn_like(y)
        flops = 2.0 * N * (H // s) * (W // s) * co * ci * R * R
        ours = {
            "fprop": timeit(lambda: C.conv_fprop(x, w, s, pad), args.iters, flush),
            "dgrad": timeit(lambda: C.conv_dgrad(dy, w, x.shape, s, pad), args.iters, flush),
            "wgrad": timeit(lambda: C.conv_wgrad(dy, x, w, s, pad), args.iters, flush),
        }
        if args.ours_only:
            print(json.dumps({"shape": f"N{N} {ci}x{H}x{W} -> {co} k{R} s{s}", "ours_us": ours}), flush=True)
            continue
        xg = x.detach().clone().requires_grad_(True)
        wg = w.detach().clone().requires_grad_(True)
        yc = F.conv2d(xg, wg, None, s, pad)
        lib = {
            "fprop": timeit(lambda: F.conv2d(x, w, None, s, pad), args.iters, flush),
            "dgrad": timeit(lambda: torch.autograd.grad(yc, xg, dy, retain_graph=True), args.iters, flush),
            "wgrad": timeit(lambda: torch.autograd.grad(yc, wg, dy, retain_graph=True), args.iters, flush),
        }
        row = {"shape": f"N{N} {ci}x{H}x{W} -> {co} k{R} s{s}", "gflop": round(flops / 1e9, 1)}
        for k in ("fprop", "dgrad", "wgrad"):
            row[k] = {"ours_us": round(ours[k], 1), "cudnn_us": round(lib[k], 1),
                      "ours_tflops": round(flops / ours[k] / 1e6, 1),
                      "frac_of_measured_peak": round(flops / ours[k] / 1e6 / peak, 3),
                      "speedup_vs_cudnn": round(lib[k] / ours[k], 2)}
        rows.append(row)
        print(json.dumps(row), flush=True)
        del x, w, y, dy, xg, wg, yc
    if args.ours_only:
        return
    tot_o = sum(r[k]["ours_us"] for r in rows for k in ("fprop", "dgrad", "wgrad"))
    tot_c = sum(r[k]["cudnn_us"] for r in rows for k in ("fprop", "dgrad", "wgrad"))
    summary = {"total_ours_us": round(tot_o, 1), "total_cudnn_us": round(tot_c, 1), "peak_tflops": peak}
    print(json.dumps(summary), flush=True)
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        json.dump({"rows": rows, "summary": summary}, open(args.out, "w"), indent=1)


if __name__ == "__main__":
    main()
