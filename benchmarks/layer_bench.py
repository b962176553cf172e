#!/usr/bin/env python
"""Per-layer roofline table for every convolution of ResNet-50 (batch 256, 224x224, bf16 NHWC) on this
repo's kernels: forward (with the BN statistics in the epilogue), dgrad, wgrad — time, achieved GB/s and
TFLOP/s, and the fraction of the slower of the two rooflines (MEASURED_PEAKS.json: HBM copy GB/s, cuBLAS
bf16 TFLOP/s burst).  CUDA events, 3 warm-ups, L2 flushed before each timed call, median of --iters.

    python benchmarks/layer_bench.py [--batch 256] [--iters 7] [--out layer_bench.json]
"""
import argparse, collections, json, os, sys
import torch
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
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--iters", type=int, default=7)
    ap.add_argument("--out", default=None, help="also write the rows to this JSON file")
    args = ap.parse_args()
    from distributed_torch_horovod_gcp_b200.models import resnet50
    from distributed_torch_horovod_gcp_b200.ops import kernels, conv as CV
    assert kernels.has("conv_implicit_gemm")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    hbm, tf = 3350.0, 989.0      # H100 SXM data sheet (not measured); MEASURED_PEAKS.json overrides
    try:
        pk = json.load(open(os.path.join(root, "MEASURED_PEAKS.json")))
        hbm, tf = pk["hbm_gbs"], pk["bf16_tflops"]
    except Exception:
        pass
    dev = torch.device("cuda")
    model = resnet50().to(dev).to(torch.bfloat16).to(memory_format=torch.channels_last)
    shapes = collections.OrderedDict()
    hooks = []
    for name, m in model.named_modules():
        if isinstance(m, torch.nn.Conv2d):
            def hook(mod, inp, out, name=name):
                key = (mod.in_channels, mod.out_channels, mod.kernel_size[0], mod.stride[0], tuple(inp[0].shape[2:]))
                shapes.setdefault(key, [mod, 0])[1] += 1
            hooks.append(m.register_forward_hook(hook))
    # conv modules are called through ops.functional, not Module.__call__: enumerate from a trace instead
    for h in hooks:
        h.remove()
    H = 224
    layers = []     # (name, module, input HxW)
    hw = H // 2
    layers.append(("conv1", model.conv1, H))
    hw = hw // 2
    for li, layer in enumerate([model.layer1, model.layer2, model.layer3, model.layer4]):
        for bi, blk in enumerate(layer):
            s = blk.conv2.stride[0]
            layers.append((f"layer{li + 1}.{bi}.conv1", blk.conv1, hw))
            layers.append((f"layer{li + 1}.{bi}.conv2", blk.conv2, hw))
            if blk.downsample is not None:
                layers.append((f"layer{li + 1}.{bi}.downsample", blk.downsample[0], hw))
            hw = hw // s
            layers.append((f"layer{li + 1}.{bi}.conv3", blk.conv3, hw))
    uniq = collections.OrderedDict()
    for name, m, size in layers:
        key = (m.in_channels, m.out_channels, m.kernel_size[0], m.stride[0], size)
        if key in uniq:
            uniq[key][2] += 1
        else:
            uniq[key] = [name, m, 1]
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    N = args.batch
    rows = []
    tot = collections.Counter()
    for (ci, co, k, s, size), (name, conv, count) in uniq.items():
        x = torch.randn(N, ci, size, size, device=dev).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
        x.requires_grad_(ci != 3)
        w = conv.weight
        stats = torch.zeros(2 * co, dtype=torch.float32, device=dev)
        def fwd():
            stats.zero_()
            return CV.conv2d(x, conv, stats=stats)
        y = fwd()
        dy = torch.randn_like(y)
        oh = y.shape[2]
        flops = 2.0 * N * oh * oh * co * ci * k * k
        act_in, act_out = x.numel() * 2, y.numel() * 2
        t_f = timeit(fwd, args.iters, flush)
        res = {"fwd": (t_f, act_in + act_out)}
        if ci != 3:
            t_d = timeit(lambda: torch.autograd.grad(y, x, dy, retain_graph=True), args.iters, flush)
            res["dgrad"] = (t_d, act_in + act_out)
        t_w = timeit(lambda: torch.autograd.grad(y, w, dy, retain_graph=True), args.iters, flush)
        res["wgrad"] = (t_w, act_in + act_out)
        row = {"layer": name, "x": f"{ci}x{size}x{size}", "cout": co, "k": k, "stride": s, "count": count,
               "gflop": round(flops / 1e9, 1)}
        for kind, (t, nbytes) in res.items():
            ideal = max(nbytes / (hbm * 1e3), flops / (tf * 1e6))       # us
            row[kind] = {"us": round(t, 1), "gbs": round(nbytes / t / 1e3, 0), "tflops": round(flops / t / 1e6, 0),
                         "frac_of_roofline": round(ideal / t, 2)}
            tot[kind] += t * count
            tot[kind + "_ideal"] += ideal * count
        rows.append(row)
        print(json.dumps(row), flush=True)
        del x, y, dy
    summary = {k: round(v, 1) for k, v in tot.items()}
    summary["peaks"] = {"hbm_gbs": hbm, "bf16_tflops": tf}
    print(json.dumps(summary), flush=True)
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        json.dump({"rows": rows, "summary": summary}, open(args.out, "w"), indent=1)


if __name__ == "__main__":
    main()
