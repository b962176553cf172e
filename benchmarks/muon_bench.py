"""Cost of Muon in the fused engine on GPT-2 small (124M), bf16, one GPU, B = 8, S = 1024.

Four arms, built in this one process and timed in alternating rounds with CUDA events, so they see the same
clocks and neighbours:
- ``adamw``: the training script's ``gpt_optimizer`` (AdamW, betas (0.9, 0.95), wd 0.1 on matrices and
  embeddings), fused engine, whole step captured as a CUDA graph;
- ``muon``: ``gpt_muon_optimizer`` (``hvd.Muon`` on the blocks' qkv / proj / fc1 / fc2 weights with
  ``adjust_lr_fn="match_rms_adamw"``, AdamW on the rest), fused engine, CUDA graph;
- ``muon_eager``: the fused ``muon`` arm's engine run without a graph, so the host work of its hooks (three
  ``ops.gemm.gemm`` calls per matrix and iteration) is in the step;
- ``muon_generic``: the same optimizer with ``DistributedOptimizer(fused=False)``: the all-reduce, then the
  eager ``step()`` after backward.  Its AdamW groups count steps on the host, so it runs eagerly, not graphed.
Separately, on the engine's side stream: the Newton–Schulz GEMMs of every Muon bucket, and the reduce (K12),
normalise (K13) and apply (K14) kernels of every Muon bucket, each phase alone.  These extra launches reduce zero
gradients and move the parameters; only their times are read.  Prints one JSON line with the card name and power
limit read in the same run.

    python benchmarks/muon_bench.py [--iters 10] [--rounds 5]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "app"))
os.environ.setdefault("B200DP_FUSED_SINGLE", "1")
os.environ.setdefault("B200DP_OFFLINE", "1")

import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True)
    name, power = [s.strip() for s in q.stdout.splitlines()[0].split(",")]
    return name, power


def make_arm(hvd, arm, x, y):
    import torch_train
    from distributed_torch_horovod_gcp_b200.models import gpt2
    from distributed_torch_horovod_gcp_b200.utils.graph import GraphedStep
    torch.manual_seed(0)
    model = gpt2().cuda().to(torch.bfloat16)
    base = torch_train.gpt_optimizer(model, 6e-4) if arm == "adamw" else torch_train.gpt_muon_optimizer(model, 6e-4)
    opt = hvd.DistributedOptimizer(base, named_parameters=model.named_parameters(), fused=arm != "muon_generic")
    if (opt.fused_engine is None) != (arm == "muon_generic"):
        raise RuntimeError(f"{arm}: the fused engine did not engage as expected")

    def step(xb, yb):
        loss = F.cross_entropy(model(xb).float(), yb)
        loss.backward()
        opt.step()
        opt.zero_grad()
        return loss.detach()

    run = step if arm in ("muon_generic", "muon_eager") else GraphedStep(step, [x, y], warmup=3)
    return {"run": run, "opt": opt, "model": model}


def time_steps(arm, x, y, iters):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        arm["run"](x, y)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def time_ns(arm, iters):
    """Device time of one step's Newton–Schulz GEMMs (every matrix of every Muon bucket) on the side stream."""
    eng = arm["opt"].fused_engine
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    with torch.cuda.stream(eng.side):
        e0.record(eng.side)
        for _ in range(iters):
            for b in eng.buckets:
                if b.index in eng._mu_args:
                    eng._newton_schulz(b, eng.opt.param_groups[b.group_index])
        e1.record(eng.side)
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def time_muon_kernels(arm, iters):
    """Device time of each Muon phase kernel alone, over every Muon bucket, on the side stream: {phase: ms}."""
    eng = arm["opt"].fused_engine
    S, out = eng.S, {}
    for name, phase in (("k12_reduce", S.MUON_REDUCE), ("k13_normalize", S.MUON_NORMALIZE),
                        ("k14_apply", S.MUON_APPLY)):
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(eng.side)
        for _ in range(iters):
            for b in eng.buckets:
                if b.index in eng._mu_args:
                    eng.symm.launch_bucket("muon", eng._args[b.index], eng._mu_args[b.index], phase,
                                           eng._kdtype[b.index], eng._kbytes[b.index], eng.side)
        e1.record(eng.side)
        torch.cuda.synchronize()
        out[name] = round(e0.elapsed_time(e1) / iters, 4)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10, help="steps per timed round")
    ap.add_argument("--rounds", type=int, default=5, help="alternating rounds per arm")
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--seq", type=int, default=1024)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        print(json.dumps({"error": "muon_bench.py needs a CUDA device"}))
        return 1
    import distributed_torch_horovod_gcp_b200.torch as hvd
    hvd.init()
    torch.cuda.set_device(0)
    name, power = card()
    torch.manual_seed(1)
    x = torch.randint(0, 50257, (args.batch, args.seq), device="cuda")
    y = torch.randint(0, 50257, (args.batch * args.seq,), device="cuda")
    keys = ("adamw", "muon", "muon_eager", "muon_generic")
    arms = {k: make_arm(hvd, k, x, y) for k in keys}
    for arm in arms.values():
        time_steps(arm, x, y, 2)                      # warm every arm before the timed rounds
    ms = {k: [] for k in keys}
    for _ in range(args.rounds):
        for k in keys:
            ms[k].append(time_steps(arms[k], x, y, args.iters))
    eng = arms["muon"]["opt"].fused_engine
    med = {k: statistics.median(v) for k, v in ms.items()}
    print(json.dumps({
        "model": "gpt2", "dtype": "bf16", "batch": args.batch, "seq": args.seq, "gpu": name, "power_limit": power,
        "muon_matrices": sum(len(eng._mu_mats[i]) for i in eng._mu_args), "muon_buckets": len(eng._mu_args),
        **{f"ms_per_step_{k}": round(med[k], 3) for k in keys},
        "muon_vs_adamw": round(med["muon"] / med["adamw"], 4),
        "muon_generic_vs_muon": round(med["muon_generic"] / med["muon"], 4),
        "muon_eager_minus_graphed_ms": round(med["muon_eager"] - med["muon"], 3),
        "ns_ms_per_step": round(time_ns(arms["muon"], args.iters), 3),
        "muon_kernels_ms_per_step": time_muon_kernels(arms["muon"], args.iters),
        **{f"rounds_{k}": [round(v, 3) for v in ms[k]] for k in keys}}), flush=True)
    hvd.shutdown()
    return 0


if __name__ == "__main__":
    sys.exit(main())
