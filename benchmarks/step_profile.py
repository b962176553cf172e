#!/usr/bin/env python
"""Per-kernel-family share of the benchmark's training step: ResNet-50, batch 256, bf16, NHWC, one GPU, the
step captured in a CUDA graph exactly as bench.py builds it.  A few replays are traced with torch.profiler
(CUDA activities); the trace goes to --out-dir and the GPU time of each kernel family is printed per step and
as a share of all kernel time.

Families: conv_bf16_kernel<BN,MODE> (MODE 0 fprop, 1 dgrad, 2 wgrad), gemm_bf16_kernel<BN,A_MN,B_MN>, the
BatchNorm kernels, the gradient-communication / optimizer-update kernels, other kernels of this project, and
ATen / vendor-library glue.

    python benchmarks/step_profile.py [--steps 5] [--warmup 5] [--out-dir DIR]
"""
import argparse, collections, json, os, re, sys, tempfile
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

_TEMPLATED = re.compile(r"(conv_bf16_kernel|gemm_bf16_kernel)<([^>]*)>")
_BN = re.compile(r"(^|[^a-z])(bn|batch_?norm)", re.I)
_COMM = re.compile(r"allreduce|reduce_scatter|allgather|broadcast|fused_|sgd|update|cast_acc|comm", re.I)
_ATEN = re.compile(r"at::|at_cuda|cudnn|cublas|cutlass|sm90_xmma|nvjet|void (elementwise|vectorized|reduce)_", re.I)


def family(name: str) -> str:
    m = _TEMPLATED.search(name)
    if m:
        args = ",".join(a.strip() for a in m.group(2).split(","))
        return f"{m.group(1)}<{args}>"
    if _ATEN.search(name):
        return "ATen / library glue"
    if _BN.search(name):
        return "BatchNorm kernels"
    if _COMM.search(name):
        return "comm / update kernels"
    return "other own kernels"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5, help="graph replays traced")
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--out-dir", default=os.path.join(tempfile.gettempdir(), "step_profile"),
                    help="trace and JSON summary go here")
    args = ap.parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile
    import bench
    import distributed_torch_horovod_gcp_b200.torch as hvd
    from distributed_torch_horovod_gcp_b200.utils.graph import GraphedStep

    assert torch.cuda.is_available(), "step_profile.py needs a CUDA device"
    hvd.init()
    torch.cuda.set_device(0)
    dev = torch.device("cuda", 0)
    argv, sys.argv = sys.argv, sys.argv[:1]
    bargs = bench.parse()                       # bench.py's defaults: resnet50, bf16, 224x224
    sys.argv = argv
    bargs.batch = args.batch
    wl = bench.Workload(bargs, dev, 0)
    model = wl.build_model()
    os.environ.setdefault("B200DP_FUSED_SINGLE", "1")
    opt = hvd.DistributedOptimizer(wl.build_optimizer(model), named_parameters=model.named_parameters())
    hvd.broadcast_parameters(model.state_dict(), root_rank=0)
    data = wl.data()
    batches = [data.next() for _ in range(2)]

    def eager_step(x, y):
        loss = wl.loss(model(x), y)
        loss.backward()
        opt.step()
        opt.zero_grad(set_to_none=False)
        return loss.detach()

    step = GraphedStep(eager_step, list(batches[0]), warmup=3)
    for i in range(args.warmup):
        step(*batches[i % 2])
    torch.cuda.synchronize()

    os.makedirs(args.out_dir, exist_ok=True)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for i in range(args.steps):
            step(*batches[i % 2])
        torch.cuda.synchronize()
    prof.export_chrome_trace(os.path.join(args.out_dir, "step.pt.trace.json"))

    per = collections.Counter()
    calls = collections.Counter()
    for ev in prof.key_averages():
        t = getattr(ev, "device_time_total", None)
        if t is None:
            t = ev.cuda_time_total
        if t <= 0 or ev.key.startswith("ProfilerStep") or "graphed_step" in ev.key or "Memcpy" in ev.key \
                or "Memset" in ev.key:
            continue
        f = family(ev.key)
        per[f] += t
        calls[f] += ev.count
    total = sum(per.values())
    props = torch.cuda.get_device_properties(dev)
    rows = [{"family": f, "ms_per_step": round(t / 1e3 / args.steps, 3), "share": round(t / total, 4),
             "launches_per_step": calls[f] // args.steps} for f, t in per.most_common()]
    print(f"device: {props.name}; kernel time per step {total / 1e3 / args.steps:.2f} ms over {args.steps} replays")
    print(f"{'family':44s} {'ms/step':>9s} {'share':>7s} {'launches':>9s}")
    for r in rows:
        print(f"{r['family']:44s} {r['ms_per_step']:9.3f} {100 * r['share']:6.1f}% {r['launches_per_step']:9d}")
    with open(os.path.join(args.out_dir, "step_profile.json"), "w") as fh:
        json.dump({"device": props.name, "kernel_ms_per_step": round(total / 1e3 / args.steps, 3), "families": rows},
                  fh, indent=1)
    hvd.shutdown()


if __name__ == "__main__":
    main()
