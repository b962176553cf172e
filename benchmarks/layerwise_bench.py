"""Cost of LARS / LAMB in the fused engine (``hvd.LARS`` / ``hvd.LAMB`` under ``DistributedOptimizer``), one GPU.

Each config compares the optimizer a user would otherwise train with against its layer-wise counterpart:
ResNet-50 bf16 channels_last at batch 256 (224x224): SGD momentum 0.9, wd 1e-4 vs LARS; ViT-B/16 bf16 (224x224):
AdamW vs LAMB.  Both arms are captured as whole-step CUDA graphs and replayed in alternating rounds in this one
process, each round timed with CUDA events, so both see the same clocks and neighbours.  Separately, each arm's
per-bucket optimizer kernels are timed alone on the engine's side stream: the one-shot fused kernel (K1) of the
baseline arm, and the reduce + direction (K10) and ratio + update (K11) phases of the layer-wise arm.  These
extra launches reduce zero gradients and move the parameters; the benchmark only reads the times.  Biases and
norm-layer parameters go in a group with ``weight_decay=0, adaptive=False`` in the layer-wise arms.  Prints one
JSON line per config with the card name and power limit read in the same run.

    python benchmarks/layerwise_bench.py [--configs resnet50,vit_b_16] [--iters 20] [--rounds 5]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
os.environ.setdefault("B200DP_FUSED_SINGLE", "1")

import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True)
    name, power = [s.strip() for s in q.stdout.splitlines()[0].split(",")]
    return name, power


def _groups(model, wd):
    return [{"params": [p for p in model.parameters() if p.dim() > 1], "weight_decay": wd},
            {"params": [p for p in model.parameters() if p.dim() <= 1], "weight_decay": 0.0, "adaptive": False}]


def build(hvd, cfg, arm, dev, batch):
    """(model, torch optimizer, example inputs, loss) for one arm; the same seed for both arms."""
    from distributed_torch_horovod_gcp_b200.models import build as build_model
    torch.manual_seed(0)
    model = build_model(cfg, num_classes=1000).to(dev).to(torch.bfloat16)
    if cfg == "resnet50":
        model = model.to(memory_format=torch.channels_last)
        opt = torch.optim.SGD(model.parameters(), lr=0.1, momentum=0.9, weight_decay=1e-4) if arm == "base" else \
            hvd.LARS(_groups(model, 1e-4), lr=0.1, momentum=0.9)
    else:
        opt = torch.optim.AdamW(model.parameters(), lr=1e-3, weight_decay=0.05) if arm == "base" else \
            hvd.LAMB(_groups(model, 0.05), lr=1e-3)
    model.train()
    x = torch.randn(batch, 3, 224, 224, device=dev, dtype=torch.bfloat16)
    if cfg == "resnet50":
        x = x.contiguous(memory_format=torch.channels_last)
    y = torch.randint(0, 1000, (batch,), device=dev)
    return model, opt, (x, y), lambda out, t: F.cross_entropy(out.float(), t)


def make_arm(hvd, cfg, arm, dev, batch):
    from distributed_torch_horovod_gcp_b200.utils.graph import GraphedStep
    model, base, inputs, loss_fn = build(hvd, cfg, arm, dev, batch)
    opt = hvd.DistributedOptimizer(base, named_parameters=model.named_parameters())
    if opt.fused_engine is None:
        raise RuntimeError("the fused engine is not available: this benchmark measures it")

    def step(x, y):
        loss = loss_fn(model(x), y)
        loss.backward()
        opt.step()
        opt.zero_grad()
        return loss.detach()

    g = GraphedStep(step, list(inputs), warmup=3)
    return {"graph": g, "inputs": inputs, "opt": opt, "model": model}


def time_replays(arm, iters):
    g, (x, y) = arm["graph"], arm["inputs"]
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        g(x, y)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def time_kernels(arm, iters):
    """Device time of every bucket's optimizer kernels alone on the side stream, with the argument blocks the
    graph's last capture left behind: {"k1": ms} for the baseline arm, {"k10": ms, "k11": ms, "total": ms}
    for the layer-wise arm."""
    eng = arm["opt"].fused_engine
    S, symm = eng.S, eng.symm

    def run(phases):
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(eng.side)
        for _ in range(iters):
            for b in eng.buckets:
                a, nbytes = eng._args[b.index], b.nbytes
                for ph in phases:
                    if ph is None:
                        symm.launch_allreduce(a, eng._algo[b.index], b.dtype, nbytes, eng.side)
                    else:
                        symm.launch_bucket("lw", a, eng._lw_args[b.index], ph, b.dtype, nbytes, eng.side)
        e1.record(eng.side)
        torch.cuda.synchronize()
        return round(e0.elapsed_time(e1) / iters, 4)

    if not eng.layerwise:
        return {"k1": run([None])}
    # K11 alone re-applies the R the last K10 left; timing each phase on its own isolates its cost
    return {"k10": run([S.LW_REDUCE]), "k11": run([S.LW_APPLY]), "total": run([S.LW_REDUCE, S.LW_APPLY])}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", default="resnet50,vit_b_16")
    ap.add_argument("--iters", type=int, default=20, help="graph replays per timed round")
    ap.add_argument("--rounds", type=int, default=5, help="alternating rounds per arm")
    ap.add_argument("--resnet-batch", type=int, default=256)
    ap.add_argument("--vit-batch", type=int, default=128)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        print(json.dumps({"error": "layerwise_bench.py needs a CUDA device"}))
        return 1
    import distributed_torch_horovod_gcp_b200.torch as hvd
    hvd.init()
    torch.cuda.set_device(0)
    dev = torch.device("cuda", 0)
    name, power = card()
    names = {"resnet50": ("sgd", "lars"), "vit_b_16": ("adamw", "lamb")}
    for cfg in args.configs.split(","):
        batch = args.resnet_batch if cfg == "resnet50" else args.vit_batch
        arms = {"base": make_arm(hvd, cfg, "base", dev, batch), "lw": make_arm(hvd, cfg, "lw", dev, batch)}
        for arm in arms.values():
            time_replays(arm, max(2, args.iters // 4))          # warm every graph before the timed rounds
        ms = {"base": [], "lw": []}
        for _ in range(args.rounds):
            for key in ("base", "lw"):
                ms[key].append(time_replays(arms[key], args.iters))
        kernels = {key: time_kernels(arm, args.iters) for key, arm in arms.items()}
        eng = arms["lw"]["opt"].fused_engine
        base, lw = statistics.median(ms["base"]), statistics.median(ms["lw"])
        b_name, l_name = names[cfg]
        print(json.dumps({
            "config": cfg, "batch": batch, "gpu": name, "power_limit": power,
            "optimizers": [b_name, l_name], "buckets": len(eng.buckets), "params": sum(b.numel for b in eng.buckets),
            "chunks": int(eng.lw_chunks.shape[0]),
            "launches_per_step": {b_name: arms["base"]["graph"].kernels_per_replay,
                                  l_name: arms["lw"]["graph"].kernels_per_replay},
            f"ms_per_step_{b_name}": round(base, 4), f"ms_per_step_{l_name}": round(lw, 4),
            "overhead_ms": round(lw - base, 4), "overhead_pct": round(100.0 * (lw - base) / base, 3),
            f"rounds_{b_name}": [round(v, 4) for v in ms["base"]], f"rounds_{l_name}": [round(v, 4) for v in ms["lw"]],
            f"optimizer_kernels_ms_{b_name}": kernels["base"], f"optimizer_kernels_ms_{l_name}": kernels["lw"]}),
            flush=True)
        del arms
        torch.cuda.empty_cache()
    hvd.shutdown()
    return 0


if __name__ == "__main__":
    sys.exit(main())
