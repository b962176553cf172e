"""Stacked / bidirectional LSTM on the K5 recurrence kernels against cuDNN's RNN, on one GPU.

For each (layers, directions, batch, steps) config, with F = 23 input features and hidden size 256, fp32:
  * ``fwd_bwd_ms``: forward + backward of the reference model's LSTM alone (upstream gradients on seq),
    device time from CUDA events over many iterations after warm-up;
  * ``step_ms``: a whole training step of the reference model (LSTM + head + MSE +
    ``DistributedOptimizer(Adam)`` with the fused engine), captured in one CUDA graph and replayed.
Both for K5 (the default path) and for cuDNN (``model._fused = False``, cuDNN's default TF32 on).
``--dropout P`` also times every config with inter-layer dropout P (``nn.LSTM(dropout=P)``, training mode;
one-layer configs have no layer to drop after and are timed at P = 0 only).
Prints one JSON line per (config, dropout) with the card name and power limit read in the same run.

    python benchmarks/lstm_bench.py [--iters 200] [--warmup 20] [--dropout 0.2]
"""
import argparse
import copy
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
os.environ.setdefault("B200DP_FUSED_SINGLE", "1")

import torch  # noqa: E402

CONFIGS = [(L, D, B, T) for (L, D) in [(1, 1), (2, 1), (1, 2), (2, 2), (4, 2)] for B in (32, 256) for T in (10, 50)]
F = 23


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


def fwd_bwd(model, x, g):
    from distributed_torch_horovod_gcp_b200.ops import functional as F2
    lstm = F2.lstm_reference if model._fused is False else F2.lstm

    def run():
        h = model.init_hidden(x.shape[0])
        seq, _ = lstm(x, model.lstm, h)
        seq.backward(g)
    return run


def graphed_step(hvd, model, x, y, warmup):
    from distributed_torch_horovod_gcp_b200.utils.graph import GraphedStep
    opt = hvd.DistributedOptimizer(torch.optim.Adam(model.parameters(), lr=1e-6),
                                   named_parameters=model.named_parameters())

    def step(xb, yb):
        loss = torch.nn.functional.mse_loss(model(xb), yb)
        loss.backward()
        opt.step()
        opt.zero_grad()
        return loss.detach()
    gs = GraphedStep(step, [x, y], warmup=warmup)
    return lambda: gs(x, y)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--dropout", type=float, default=0.0, help="also time at this inter-layer dropout")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("lstm_bench needs a GPU")
    import distributed_torch_horovod_gcp_b200.torch as hvd
    from distributed_torch_horovod_gcp_b200.models import LSTM
    from distributed_torch_horovod_gcp_b200.ops import kernels
    assert kernels.has("lstm_recurrent"), "K5 kernels are not built"
    hvd.init()
    dev = torch.device("cuda", 0)
    name, power = card()
    for (L, D, B, T), p in [(c, p) for c in CONFIGS for p in sorted({0.0, args.dropout if c[0] > 1 else 0.0})]:
        torch.manual_seed(0)
        base = LSTM(F, T, 1, 256, n_layers=L, bidirectional=D == 2, device=dev, dropout=p)
        x = torch.randn(B, T, F, device=dev)
        y = torch.randn(B, 1, 1, device=dev)
        g = torch.randn(B, T, D * 256, device=dev)
        res = {"layers": L, "directions": D, "batch": B, "steps": T, "features": F, "hidden": 256, "dropout": p}
        for arm in ("k5", "cudnn"):
            m = copy.deepcopy(base)
            m._fused = False if arm == "cudnn" else None
            res[f"{arm}_fwd_bwd_ms"] = round(time_ms(fwd_bwd(m, x, g), args.iters, args.warmup), 4)
            m = copy.deepcopy(base)
            m._fused = False if arm == "cudnn" else None
            res[f"{arm}_step_ms"] = round(time_ms(graphed_step(hvd, m, x, y, 3), args.iters, args.warmup), 4)
        res["fwd_bwd_speedup"] = round(res["cudnn_fwd_bwd_ms"] / res["k5_fwd_bwd_ms"], 3)
        res["step_speedup"] = round(res["cudnn_step_ms"] / res["k5_step_ms"], 3)
        res.update({"gpu": name, "power_limit": power, "cudnn_allow_tf32": torch.backends.cudnn.allow_tf32})
        print(json.dumps(res), flush=True)
    hvd.shutdown()


if __name__ == "__main__":
    main()
