"""Cost of clipping by global norm in the fused engine (``DistributedOptimizer(max_grad_norm=)``), one GPU.

For each config, two replicas of the same training step are captured as whole-step CUDA graphs: one without
``max_grad_norm`` (the fused one-shot kernel per bucket) and one with it (reduce into R per bucket, one
finalize launch, one update launch per bucket).  The two graphs are replayed in alternating rounds in this
one process and each round is timed with CUDA events, so both arms see the same clocks and neighbours.
Separately, the finalize + update stage of the clip arm (the part that no longer overlaps backward) is
timed alone on the engine's side stream with CUDA events.

Configs: ResNet-50 bf16 channels_last at batch 256 (224x224, SGD momentum 0.9, wd 1e-4) and the reference
LSTM config (LSTM(23 -> 256), window 10, batch 32, fp32, Adam lr 1e-6).  Prints one JSON line per config
with the card name and power limit read in the same run.

    python benchmarks/clip_bench.py [--configs resnet50,lstm] [--iters 20] [--rounds 5]
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


def build(cfg, dev, batch):
    """(model, torch optimizer, example inputs, loss) for one config; the same seed for both arms."""
    torch.manual_seed(0)
    if cfg == "lstm":
        from distributed_torch_horovod_gcp_b200.models import LSTM
        model = LSTM(n_features=23, window_size=10, output_size=1, h_size=256, device=dev).to(dev)
        opt = torch.optim.Adam(model.parameters(), lr=1e-6)
        x = torch.rand(batch, 10, 23, device=dev)
        y = torch.rand(batch, 1, 1, device=dev)
        return model, opt, (x, y), F.mse_loss
    from distributed_torch_horovod_gcp_b200.models import build as build_model
    model = build_model("resnet50", num_classes=1000).to(dev).to(torch.bfloat16)
    model = model.to(memory_format=torch.channels_last).train()
    opt = torch.optim.SGD(model.parameters(), lr=0.1, momentum=0.9, weight_decay=1e-4)
    x = torch.randn(batch, 3, 224, 224, device=dev, dtype=torch.bfloat16).contiguous(
        memory_format=torch.channels_last)
    y = torch.randint(0, 1000, (batch,), device=dev)
    return model, opt, (x, y), lambda out, t: F.cross_entropy(out.float(), t)


def make_arm(hvd, cfg, dev, batch, max_grad_norm):
    from distributed_torch_horovod_gcp_b200.utils.graph import GraphedStep
    model, base, inputs, loss_fn = build(cfg, dev, batch)
    opt = hvd.DistributedOptimizer(base, named_parameters=model.named_parameters(), max_grad_norm=max_grad_norm)
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


def time_clip_stage(arm, iters):
    """Device time of the finalize + per-bucket update launches alone, on the engine's side stream (these
    extra launches update the parameters again; the benchmark only reads the time)."""
    eng = arm["opt"].fused_engine
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(eng.side)
    for _ in range(iters):
        eng._clip_and_update()
    e1.record(eng.side)
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", default="resnet50,lstm")
    ap.add_argument("--iters", type=int, default=20, help="graph replays per timed round")
    ap.add_argument("--rounds", type=int, default=5, help="alternating rounds per arm")
    ap.add_argument("--max-grad-norm", type=float, default=1.0)
    ap.add_argument("--resnet-batch", type=int, default=256)
    ap.add_argument("--lstm-batch", type=int, default=32)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        print(json.dumps({"error": "clip_bench.py needs a CUDA device"}))
        return 1
    import distributed_torch_horovod_gcp_b200.torch as hvd
    hvd.init()
    torch.cuda.set_device(0)
    dev = torch.device("cuda", 0)
    name, power = card()
    for cfg in args.configs.split(","):
        batch = args.lstm_batch if cfg == "lstm" else args.resnet_batch
        iters = args.iters * (10 if cfg == "lstm" else 1)
        arms = {"off": make_arm(hvd, cfg, dev, batch, None), "on": make_arm(hvd, cfg, dev, batch, args.max_grad_norm)}
        for arm in arms.values():
            time_replays(arm, max(2, iters // 4))          # warm every graph before the timed rounds
        ms = {"off": [], "on": []}
        for _ in range(args.rounds):
            for key in ("off", "on"):
                ms[key].append(time_replays(arms[key], iters))
        stage = time_clip_stage(arms["on"], iters)
        eng = arms["on"]["opt"].fused_engine
        off, on = statistics.median(ms["off"]), statistics.median(ms["on"])
        print(json.dumps({
            "config": cfg, "batch": batch, "gpu": name, "power_limit": power,
            "buckets": len(eng.buckets), "params": sum(b.numel for b in eng.buckets),
            "launches_per_step": {"off": arms["off"]["graph"].kernels_per_replay,
                                  "on": arms["on"]["graph"].kernels_per_replay},
            "ms_per_step_off": round(off, 4), "ms_per_step_on": round(on, 4),
            "overhead_ms": round(on - off, 4), "overhead_pct": round(100.0 * (on - off) / off, 3),
            "rounds_off": [round(v, 4) for v in ms["off"]], "rounds_on": [round(v, 4) for v in ms["on"]],
            "finalize_apply_ms": round(stage, 4),
            "grad_norm": float(arms["on"]["opt"].grad_norm)}), flush=True)
        del arms
        torch.cuda.empty_cache()
    hvd.shutdown()
    return 0


if __name__ == "__main__":
    sys.exit(main())
