#!/usr/bin/env python
"""wgmma flash attention (csrc/attn_sm90.cu) vs F.scaled_dot_product_attention on the ViT-B/16 shape
(batch 128, 12 heads, 197 tokens, d 64) and a long-sequence shape; forward and forward+backward.
CUDA events, 3 warm-ups, L2 flush before each timed call, median of --iters."""
import argparse, json, os, sys
import torch
import torch.nn.functional as F
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def timeit(fn, iters, flush):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        flush.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); fn(); e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    ts.sort()
    return ts[len(ts) // 2] * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--out", default=None, help="also write the rows to this JSON file")
    args = ap.parse_args()
    from distributed_torch_horovod_gcp_b200.ops import kernels
    assert kernels.has("attention_fused")
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    rows = []
    for (B, H, S) in [(128, 12, 197), (8, 16, 1024), (4, 16, 4096)]:
        mats = [(torch.randn(B * S, H * 64, device="cuda") * 0.5).to(torch.bfloat16).requires_grad_(True) for _ in range(3)]
        q, k, v = [m.view(B, S, H, 64).transpose(1, 2) for m in mats]
        g = torch.randn(B, S, H, 64, device="cuda").to(torch.bfloat16).transpose(1, 2)
        flops_f = 4.0 * B * H * S * S * 64
        def ours_fb():
            o = kernels.attention_fused(q, k, v); o.backward(g)
        def lib_fb():
            o = F.scaled_dot_product_attention(q, k, v); o.backward(g)
        with torch.no_grad():
            t_of = timeit(lambda: kernels.attention_fused(q, k, v), args.iters, flush)
            t_lf = timeit(lambda: F.scaled_dot_product_attention(q, k, v), args.iters, flush)
        t_ob = timeit(ours_fb, args.iters, flush)
        t_lb = timeit(lib_fb, args.iters, flush)
        row = {"shape": f"B{B} H{H} S{S} d64", "fwd": {"ours_us": round(t_of, 1), "sdpa_us": round(t_lf, 1),
               "ours_tflops": round(flops_f / t_of / 1e6, 1), "speedup": round(t_lf / t_of, 2)},
               "fwd_bwd": {"ours_us": round(t_ob, 1), "sdpa_us": round(t_lb, 1),
                           "ours_tflops": round(3.5 * flops_f / t_ob / 1e6, 1), "speedup": round(t_lb / t_ob, 2)}}
        rows.append(row)
        print(json.dumps(row), flush=True)
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        json.dump(rows, open(args.out, "w"), indent=1)


if __name__ == "__main__":
    main()
