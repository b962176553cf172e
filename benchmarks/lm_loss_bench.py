"""The LM-head cross-entropy: fused (``linear_cross_entropy``, no [N, V] logits) against logits + cross-entropy.

Loss alone, forward + backward (dx and dW), bf16, D = 768, V = 50304, N in {8192, 16384, 32768}.  Three arms,
alternated in this process, device time from CUDA events:
  * ``fused``:   ``ops.xent.linear_cross_entropy`` (xent_fwd_kernel + finish, then per backward chunk
                 xent_grad_kernel and two GEMMs on the wgmma kernel);
  * ``kernels``: ``F2.linear`` on the wgmma GEMM, then ``F.cross_entropy(logits.float(), y)`` on ATen;
  * ``stand_in``: the same composition with ``B200DP_DISABLE_KERNELS=1`` (cuBLAS + ATen).
For each: ``*_ms``, ``*_peak_mib`` (``torch.cuda.max_memory_allocated`` above the inputs, after a reset) and
``*_tflops``: the 6 N D V FLOPs of one forward and two backward GEMMs over the time (the fused arm runs a fourth,
8 N D V in all, reported as ``fused_tflops_executed``).

Whole step: GPT-2 small at B = 8, S = 1024, one CUDA-graphed training step on the kernels with the fused
AdamW engine, the loss either as ``F.cross_entropy(model(x).float(), y)`` (``logits``) or as ``model(x, y)``
(``fused``), alternated; ``*_peak_mib`` is the peak allocation of building and capturing that arm's step.

Prints one JSON line per config with the card name and power limit read in the same run.

    python benchmarks/lm_loss_bench.py [--iters 20] [--warmup 3] [--rounds 3]
"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
os.environ.setdefault("B200DP_FUSED_SINGLE", "1")

import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

D, V = 768, 50304
LOSS_N = (8192, 16384, 32768)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True)
    name, power = [s.strip() for s in q.stdout.splitlines()[0].split(",")]
    return name, power


def time_ms(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def peak_mib(fn):
    """Peak allocation of one call of fn above what is allocated before it."""
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    fn()
    torch.cuda.synchronize()
    return round((torch.cuda.max_memory_allocated() - base) / 2 ** 20, 1)


class kernels_off:
    def __enter__(self):
        self.old = os.environ.get("B200DP_DISABLE_KERNELS")
        os.environ["B200DP_DISABLE_KERNELS"] = "1"

    def __exit__(self, *exc):
        if self.old is None:
            os.environ.pop("B200DP_DISABLE_KERNELS", None)
        else:
            os.environ["B200DP_DISABLE_KERNELS"] = self.old


def loss_configs(args, name, power):
    from distributed_torch_horovod_gcp_b200.ops import functional as F2
    from distributed_torch_horovod_gcp_b200.ops import xent
    for N in LOSS_N:
        g = torch.Generator(device="cuda").manual_seed(N)
        x = torch.randn(N, D, generator=g, device="cuda").bfloat16().requires_grad_(True)
        w = (torch.randn(V, D, generator=g, device="cuda") * 0.02).bfloat16().requires_grad_(True)
        y = torch.randint(0, 50257, (N,), generator=g, device="cuda")

        def fused():
            xent.linear_cross_entropy(x, w, y).backward()

        def kernels():
            F.cross_entropy(F2.linear(x, w).float(), y).backward()

        def stand_in():
            with kernels_off():
                F.cross_entropy(F2.linear(x, w).float(), y).backward()

        arms = {"fused": fused, "kernels": kernels, "stand_in": stand_in}
        res = {"config": "lm_loss", "N": N, "D": D, "V": V, "dtype": "bf16", "rounds": args.rounds,
               "iters": args.iters}
        for arm, fn in arms.items():
            x.grad = w.grad = None
            fn()                                         # .grad exists, so the peak counts only the step
            res[f"{arm}_peak_mib"] = peak_mib(fn)
        times = {a: [] for a in arms}
        for _ in range(args.rounds):
            for arm, fn in arms.items():
                times[arm].append(time_ms(fn, args.iters, args.warmup))
        flops = 6 * N * D * V
        for arm, ts in times.items():
            best = min(ts)
            res[f"{arm}_ms"] = round(best, 3)
            res[f"{arm}_ms_all"] = [round(t, 3) for t in ts]
            res[f"{arm}_tflops"] = round(flops / (best * 1e-3) / 1e12, 1)
        res["fused_tflops_executed"] = round(8 * N * D * V / (res["fused_ms"] * 1e-3) / 1e12, 1)
        res["fused_vs_kernels"] = round(res["kernels_ms"] / res["fused_ms"], 3)
        res["fused_vs_stand_in"] = round(res["stand_in_ms"] / res["fused_ms"], 3)
        res.update({"gpu": name, "power_limit": power})
        print(json.dumps(res), flush=True)
        del x, w, y
        torch.cuda.empty_cache()


def step_arm(hvd, fused_loss, x, y, warmup):
    from distributed_torch_horovod_gcp_b200.models import gpt2
    from distributed_torch_horovod_gcp_b200.utils.graph import GraphedStep
    torch.manual_seed(0)
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    model = gpt2().cuda().to(torch.bfloat16)
    groups = [{"params": [p for p in model.parameters() if p.dim() >= 2], "weight_decay": 0.1},
              {"params": [p for p in model.parameters() if p.dim() < 2], "weight_decay": 0.0}]
    opt = hvd.DistributedOptimizer(torch.optim.AdamW(groups, lr=6e-4, betas=(0.9, 0.95)),
                                   named_parameters=model.named_parameters())
    assert opt.fused_engine is not None, "the fused optimizer engine did not engage"

    def step(xb, yb):
        loss = model(xb, yb) if fused_loss else F.cross_entropy(model(xb).float(), yb.reshape(-1))
        loss.backward()
        opt.step()
        opt.zero_grad()
        return loss.detach()

    gs = GraphedStep(step, [x, y], warmup=warmup)
    torch.cuda.synchronize()
    peak = round((torch.cuda.max_memory_allocated() - base) / 2 ** 20, 1)
    return (lambda: gs(x, y)), peak


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3, help="alternations of the arms")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("lm_loss_bench needs a GPU")
    import distributed_torch_horovod_gcp_b200.torch as hvd
    from distributed_torch_horovod_gcp_b200.ops import counters, kernels
    assert kernels.has("linear_cross_entropy") and kernels.has("linear"), "the sm_90a kernels are not built"
    hvd.init()
    name, power = card()
    loss_configs(args, name, power)

    B, S = 8, 1024
    g = torch.Generator(device="cuda").manual_seed(0)
    tok = torch.randint(0, 50257, (B, S + 1), generator=g, device="cuda")
    x, y = tok[:, :-1].contiguous(), tok[:, 1:].contiguous()
    run_l, peak_l = step_arm(hvd, False, x, y, 3)
    c0 = counters.snapshot().get("xent_fwd", 0)
    run_f, peak_f = step_arm(hvd, True, x, y, 3)
    assert counters.snapshot().get("xent_fwd", 0) > c0, "the fused arm did not run the xent kernels"
    times = {"logits": [], "fused": []}
    for _ in range(args.rounds):
        times["logits"].append(time_ms(run_l, args.iters, args.warmup))
        times["fused"].append(time_ms(run_f, args.iters, args.warmup))
    res = {"config": "gpt2_step_loss", "batch": B, "seq": S, "dtype": "bf16", "rounds": args.rounds,
           "iters": args.iters, "logits_peak_mib": peak_l, "fused_peak_mib": peak_f}
    for arm, ts in times.items():
        res[f"{arm}_step_ms"] = round(min(ts), 3)
        res[f"{arm}_step_ms_all"] = [round(t, 3) for t in ts]
    res["fused_vs_logits"] = round(res["logits_step_ms"] / res["fused_step_ms"], 3)
    res.update({"gpu": name, "power_limit": power})
    print(json.dumps(res), flush=True)
    hvd.shutdown()


if __name__ == "__main__":
    main()
