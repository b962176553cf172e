"""Causal flash attention and the GPT-2 small training step, on one GPU.

Attention alone (bf16, head dim 64, B = 8 x H = 12 = 96 heads, q / k / v / dO in the model's [B, S, H, 64]
layout), forward + backward per call, device time from CUDA events over many iterations after warm-up:
  * ``causal_ms`` / ``noncausal_ms``: the kernel (``attention_fused``) with and without the causal mask;
  * ``sdpa_causal_ms``: ``F.scaled_dot_product_attention(is_causal=True)`` (PyTorch's flash kernel) on the
    same tensors;
  * ``causal_tflops``: causal fwd + bwd FLOPs, 3.5 x the forward's 4 B H S^2 64 / 2 (the backward's five
    matmuls against the forward's two), over ``causal_ms``.

Whole step: GPT-2 small (124M) in bf16 at B = 8, S = 1024, one CUDA-graphed training step (forward,
cross-entropy, backward, ``DistributedOptimizer(AdamW)`` on the fused engine).  Two arms, alternated in this
process: ``kernels`` (the sm_90a GEMM / LayerNorm / causal attention kernels) and ``stand_in``
(``B200DP_DISABLE_KERNELS=1`` during capture: cuBLAS + PyTorch LayerNorm + SDPA flash, the same fused
optimizer).  ``mfu_whole_program`` is the model FLOPs (6 N tokens, N = parameters less the position
embedding, plus causal attention 6 L B S^2 D) per step time over the 989 TFLOP/s BF16 data-sheet figure: a
whole-program rate, not any kernel's share of peak.

Dropout arm (``--dropout P``, off by default): attention adds ``causal_drop_ms`` / ``noncausal_drop_ms`` (the
kernel with ``dropout_p = P``) and ``sdpa_causal_drop_ms`` (SDPA flash with ``dropout_p = P``) on the same
tensors, and the whole step adds a third alternated arm, ``kernels_dropout``: GPT-2 small built with
``dropout = P`` (embedding, attention and residual dropout) on the kernels.

Prints one JSON line per config with the card name and power limit read in the same run.

    python benchmarks/gpt_bench.py [--iters 50] [--warmup 10] [--rounds 3] [--dropout 0.1]
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

PEAK_BF16 = 989e12
ATTN_S = (1024, 2048, 4096)


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


def attention_configs(args, name, power):
    from distributed_torch_horovod_gcp_b200.ops import attention
    B, H = 8, 12
    for S in ATTN_S:
        g = torch.Generator(device="cuda").manual_seed(S)
        q, k, v, do = [torch.randn(B, S, H, 64, generator=g, device="cuda").bfloat16().transpose(1, 2)
                       for _ in range(4)]
        q, k, v = [t.requires_grad_(True) for t in (q, k, v)]

        def kernel(causal, p=0.0):
            def run():
                attention.attention_fused(q, k, v, causal=causal, dropout_p=p).backward(do)
            return run

        def sdpa(p=0.0):
            def run():
                F.scaled_dot_product_attention(q, k, v, dropout_p=p, is_causal=True).backward(do)
            return run

        res = {"config": "attention", "batch_heads": B * H, "seq": S, "head_dim": 64}
        res["causal_ms"] = round(time_ms(kernel(True), args.iters, args.warmup), 4)
        res["noncausal_ms"] = round(time_ms(kernel(False), args.iters, args.warmup), 4)
        res["sdpa_causal_ms"] = round(time_ms(sdpa(), args.iters, args.warmup), 4)
        res["causal_vs_noncausal"] = round(res["noncausal_ms"] / res["causal_ms"], 3)
        res["causal_vs_sdpa"] = round(res["sdpa_causal_ms"] / res["causal_ms"], 3)
        flops = 3.5 * 4 * B * H * S * S * 64 / 2
        res["causal_tflops"] = round(flops / (res["causal_ms"] * 1e-3) / 1e12, 1)
        if args.dropout:
            res["dropout_p"] = args.dropout
            res["causal_drop_ms"] = round(time_ms(kernel(True, args.dropout), args.iters, args.warmup), 4)
            res["noncausal_drop_ms"] = round(time_ms(kernel(False, args.dropout), args.iters, args.warmup), 4)
            res["sdpa_causal_drop_ms"] = round(time_ms(sdpa(args.dropout), args.iters, args.warmup), 4)
            res["causal_drop_cost"] = round(res["causal_drop_ms"] / res["causal_ms"], 3)
            res["noncausal_drop_cost"] = round(res["noncausal_drop_ms"] / res["noncausal_ms"], 3)
        res.update({"gpu": name, "power_limit": power})
        print(json.dumps(res), flush=True)


def step_arm(hvd, kernels_on, x, y, warmup, dropout=0.0):
    from distributed_torch_horovod_gcp_b200.models import gpt2
    from distributed_torch_horovod_gcp_b200.utils.graph import GraphedStep
    torch.manual_seed(0)
    model = gpt2(dropout=dropout).cuda().to(torch.bfloat16)
    groups = [{"params": [p for p in model.parameters() if p.dim() >= 2], "weight_decay": 0.1},
              {"params": [p for p in model.parameters() if p.dim() < 2], "weight_decay": 0.0}]
    opt = hvd.DistributedOptimizer(torch.optim.AdamW(groups, lr=6e-4, betas=(0.9, 0.95)),
                                   named_parameters=model.named_parameters())
    assert opt.fused_engine is not None, "the fused optimizer engine did not engage"

    def step(xb, yb):
        loss = F.cross_entropy(model(xb).float(), yb)
        loss.backward()
        opt.step()
        opt.zero_grad()
        return loss.detach()

    old = os.environ.pop("B200DP_DISABLE_KERNELS", None)
    if not kernels_on:
        os.environ["B200DP_DISABLE_KERNELS"] = "1"
    try:
        gs = GraphedStep(step, [x, y], warmup=warmup)
    finally:
        os.environ.pop("B200DP_DISABLE_KERNELS", None)
        if old is not None:
            os.environ["B200DP_DISABLE_KERNELS"] = old
    n = sum(p.numel() for p in model.parameters()) - model.wpe.weight.numel()
    return (lambda: gs(x, y)), n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3, help="alternations of the whole-step arms")
    ap.add_argument("--dropout", type=float, default=0.0, help="add the dropout arms with this probability")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("gpt_bench needs a GPU")
    import distributed_torch_horovod_gcp_b200.torch as hvd
    from distributed_torch_horovod_gcp_b200.ops import counters, kernels
    assert kernels.has("attention_fused") and kernels.has("linear"), "the sm_90a kernels are not built"
    hvd.init()
    name, power = card()
    attention_configs(args, name, power)

    B, S = 8, 1024
    g = torch.Generator(device="cuda").manual_seed(0)
    tok = torch.randint(0, 50257, (B, S + 1), generator=g, device="cuda")
    x, y = tok[:, :-1].contiguous(), tok[:, 1:].reshape(-1)
    c0 = counters.snapshot()
    run_k, n_params = step_arm(hvd, True, x, y, 3)
    c1 = counters.snapshot()
    assert c1.get("attn_fwd", 0) > c0.get("attn_fwd", 0), "the kernel arm did not run the attention kernel"
    run_s, _ = step_arm(hvd, False, x, y, 3)
    assert counters.snapshot().get("attn_fwd", 0) == c1.get("attn_fwd", 0), "the stand-in arm ran a kernel"
    arms = {"kernels": run_k, "stand_in": run_s}
    if args.dropout:
        c2 = counters.snapshot()
        arms["kernels_dropout"], _ = step_arm(hvd, True, x, y, 3, args.dropout)
        assert counters.snapshot().get("attn_fwd_dropout", 0) > c2.get("attn_fwd_dropout", 0)
    times = {arm: [] for arm in arms}
    for _ in range(args.rounds):
        for arm, run in arms.items():
            times[arm].append(time_ms(run, args.iters, args.warmup))
    tokens = B * S
    flops = 6 * n_params * tokens + 6 * 12 * B * S * S * 768
    res = {"config": "gpt2_step", "batch": B, "seq": S, "dtype": "bf16", "params_counted": n_params,
           "model_flops_per_step": flops, "rounds": args.rounds, "iters": args.iters}
    for arm, ts in times.items():
        best = min(ts)
        res[f"{arm}_step_ms"] = round(best, 3)
        res[f"{arm}_step_ms_all"] = [round(t, 3) for t in ts]
        res[f"{arm}_tokens_per_s"] = round(tokens / (best * 1e-3))
        res[f"{arm}_mfu_whole_program"] = round(flops / (best * 1e-3) / PEAK_BF16, 4)
    res["speedup"] = round(res["stand_in_step_ms"] / res["kernels_step_ms"], 3)
    if args.dropout:
        res["dropout_p"] = args.dropout
        res["dropout_cost"] = round(res["kernels_dropout_step_ms"] / res["kernels_step_ms"], 3)
    res.update({"gpu": name, "power_limit": power, "peak_bf16_tflops_datasheet": PEAK_BF16 / 1e12})
    print(json.dumps(res), flush=True)
    hvd.shutdown()


if __name__ == "__main__":
    main()
