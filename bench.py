#!/usr/bin/env python
"""Headline benchmark (BASELINE.json): images/sec for ResNet-50 synthetic-ImageNet bf16
data-parallel training through ``hvd.DistributedOptimizer`` on N H100s of one node.

    python bench.py --gpus 1 --steps 20 --warmup 5
    python -m torch.distributed.run --nnodes=1 --nproc-per-node 8 --master-addr 127.0.0.1 \
        --master-port 29511 bench.py --gpus 8 --steps 20 --warmup 5
    python bench.py --model lstm           # the reference's own config: LSTM 23->256, T=10, batch 32, Adam

Prints ONE JSON line on rank 0.  ``value`` is whole-job samples/s measured on the device
(CUDA events, barrier + synchronize on both sides, max over ranks) for exactly ``--steps``
full training steps (forward, backward, gradient allreduce, optimizer update).  ``e2e`` is
the same metric through the public API with the per-step H2D copy of the inputs from pinned
host memory and a D2H read of the loss inside the timed region.

``--dump-outputs DIR`` writes what the timed path computed in its last timed step, as float32 ``.npy``
files: ``loss.npy`` (the step's loss) and ``params_sample.npy`` (the updated parameters, flattened in
``model.parameters()`` order; a fixed seeded sample of 8M elements when the model is larger).  Inputs
and initial weights are seeded, so two builds run with the same arguments can be compared output for
output.  For ResNet training the step is bit-reproducible: every cross-CTA reduction on that path
(BatchNorm statistics, split-K weight and bias gradients) sums in a fixed order.

Baselines.  ``--impl reference`` would run the unmodified reference application; it is a single
script that needs the ``horovod`` and ``GPUtil`` packages and a network download — none are
installable offline (DESIGN.md §0) — so that arm prints
``{"impl": "reference", "unavailable": ...}``.  Because of that, the default (``ours``) run ALSO
measures, in the same invocation on the same GPUs, the labelled **NCCL stand-in** (same model on
library cuDNN/cuBLAS ops + NCCL DistributedDataParallel + the stock torch optimizer — NOT
Horovod, NOT the reference) for a few steps and reports ``vs_baseline = value / stand-in`` with
``baseline_kind`` saying so; ``--impl nccl_standin`` runs only that arm.  At N > 1 the ``ours``
run additionally executes a self-check: one step through the fused sm_90a engine vs the same
step with ``torch.distributed.all_reduce`` + the torch optimizer on a cloned model, and a
cross-rank bit-equality check of the updated parameters.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)


def parse():
    p = argparse.ArgumentParser()
    p.add_argument("--gpus", type=int, default=1)
    p.add_argument("--steps", type=int, default=20)
    p.add_argument("--warmup", type=int, default=5)
    p.add_argument("--impl", default="ours", choices=["ours", "reference", "nccl_standin"])
    p.add_argument("--model", default=os.environ.get("BENCH_MODEL", "resnet50"))
    p.add_argument("--batch", type=int, default=int(os.environ.get("BENCH_BATCH", "0")),
                   help="per-GPU batch (weak scaling); default 256 (32 for lstm, the reference's value)")
    p.add_argument("--image-size", type=int, default=224)
    p.add_argument("--dtype", default=None, choices=["bf16", "fp32"])
    p.add_argument("--no-e2e", action="store_true")
    p.add_argument("--no-baseline", action="store_true", help="skip the in-run NCCL stand-in arm")
    p.add_argument("--no-selfcheck", action="store_true")
    p.add_argument("--graph", default=os.environ.get("BENCH_GRAPH", "auto"), choices=["auto", "on", "off"],
                   help="capture the whole training step (fwd+bwd+fused allreduce/update) in one CUDA "
                        "graph (ours only; 'auto' falls back to eager if capture fails)")
    p.add_argument("--lr", type=float, default=None)
    p.add_argument("--dump-outputs", default=None, metavar="DIR",
                   help="write the last timed step's loss and (sampled) updated parameters as .npy files")
    return p.parse_args()


DUMP_MAX_ELEMS = 8 << 20          # 32 MB of float32 parameters


def dump_outputs(out_dir, loss, model):
    """Loss and updated parameters of the last timed step -> DIR/loss.npy, DIR/params_sample.npy."""
    import numpy as np
    import torch
    os.makedirs(out_dir, exist_ok=True)
    np.save(os.path.join(out_dir, "loss.npy"), np.asarray([float(loss)], dtype=np.float32))
    flat = torch.cat([p.detach().reshape(-1).float() for p in model.parameters()])
    if flat.numel() > DUMP_MAX_ELEMS:
        g = torch.Generator().manual_seed(0)
        idx = torch.randperm(flat.numel(), generator=g)[:DUMP_MAX_ELEMS].sort().values
        flat = flat[idx.to(flat.device)]
    np.save(os.path.join(out_dir, "params_sample.npy"), flat.cpu().numpy())


def reference_arm(args):
    """Report why the unmodified reference application cannot run here."""
    why = None
    try:
        missing = []
        for mod in ("horovod.torch", "GPUtil"):
            try:
                __import__(mod)
            except Exception as e:  # noqa: BLE001
                missing.append(f"{mod} ({type(e).__name__})")
        if missing:
            why = ("reference is one script (no setup.py/pyproject) that imports " + ", ".join(missing) +
                   " — not installable offline; it also downloads its dataset at import time")
        else:
            why = ("reference script has no benchmark mode for BASELINE.json's metric "
                   "(ResNet-50 images/s); it only trains its LSTM on a downloaded CSV")
    except Exception as e:  # noqa: BLE001
        why = f"{type(e).__name__}: {e}"
    if int(os.environ.get("RANK", "0")) == 0:
        print(json.dumps({"impl": "reference", "unavailable": why}), flush=True)
    return 0


class Workload:
    """Model / optimizer / synthetic data for one benchmark config."""

    def __init__(self, args, dev, rank):
        import torch
        self.args, self.dev, self.rank = args, dev, rank
        self.is_lstm = args.model.lower() == "lstm"
        self.batch = args.batch or (32 if self.is_lstm else 256)
        self.dtype_name = args.dtype or ("fp32" if self.is_lstm else "bf16")
        self.dtype = torch.bfloat16 if self.dtype_name == "bf16" else torch.float32
        self.lr = args.lr if args.lr is not None else (1e-6 if self.is_lstm else 0.1)

    def build_model(self, seed=1234):
        import torch
        torch.manual_seed(seed)
        if self.is_lstm:
            from distributed_torch_horovod_gcp_b200.models import LSTM
            model = LSTM(n_features=23, window_size=10, output_size=1, h_size=256, device=self.dev)
            return model.to(self.dev)
        from distributed_torch_horovod_gcp_b200.models import build
        kw = {"num_classes": 1000}
        if "vit" in self.args.model.lower():
            kw["image_size"] = self.args.image_size
        model = build(self.args.model, **kw).to(self.dev)
        model = model.to(self.dtype).to(memory_format=torch.channels_last)
        model.train()
        return model

    def build_optimizer(self, model):
        import torch
        if self.is_lstm:       # reference: Adam(lr=1e-6), app/torch_train.py:258
            return torch.optim.Adam(model.parameters(), lr=self.lr)
        return torch.optim.SGD(model.parameters(), lr=self.lr, momentum=0.9, weight_decay=1e-4)

    def optimizer_name(self):
        return f"Adam lr={self.lr}" if self.is_lstm else "SGD momentum=0.9 wd=1e-4"

    def data(self):
        import torch
        if self.is_lstm:
            return SyntheticSeqBatches(self.batch, 10, 23, self.dev, seed=self.rank)
        from distributed_torch_horovod_gcp_b200.data import SyntheticImageBatches
        return SyntheticImageBatches(self.batch, (3, self.args.image_size, self.args.image_size), 1000,
                                     self.dev, self.dtype, ring=4, channels_last=True, seed=self.rank)

    def loss(self, out, y):
        import torch.nn.functional as F
        if self.is_lstm:
            return F.mse_loss(out, y)        # nn.MSELoss(reduction="mean"), app/torch_train.py:263
        return F.cross_entropy(out.float(), y)


class SyntheticSeqBatches:
    """Pinned-host ring of [B, T, F] windows / [B, 1, 1] targets (the reference's tensor shapes,
    app/torch_train.py:72-74,246), staged to the device per step like SyntheticImageBatches."""

    def __init__(self, batch, T, Fdim, device, ring=8, seed=0):
        import torch
        g = torch.Generator().manual_seed(seed)
        self.device = device
        self.host = [(torch.rand((batch, T, Fdim), generator=g).pin_memory(),
                      torch.rand((batch, 1, 1), generator=g).pin_memory()) for _ in range(ring)]
        self._i = 0
        self.bytes_per_batch = sum(t.numel() * t.element_size() for t in self.host[0])

    def next(self):
        x, y = self.host[self._i % len(self.host)]
        self._i += 1
        return x.to(self.device, non_blocking=True), y.to(self.device, non_blocking=True)


def run_arm(impl, wl, hvd, world, rank, steps, warmup, graph_mode, want_e2e, want_clocks, dump_dir=None):
    """Build the workload for ``impl`` and time ``steps`` training steps.  Returns a dict."""
    import torch
    from distributed_torch_horovod_gcp_b200.ops import functional as F2, counters
    from distributed_torch_horovod_gcp_b200.utils.clocks import ClockSampler
    dev = wl.dev
    F2._FORCE_REFERENCE = (impl == "nccl_standin")       # stand-in: library cuDNN/cuBLAS ops only
    model = wl.build_model()
    if impl == "nccl_standin" and wl.is_lstm:
        model._fused = False
    base = wl.build_optimizer(model)
    our_launches = lambda: 0
    eng = None
    if impl == "ours":
        os.environ.setdefault("B200DP_FUSED_SINGLE", "1")
        opt = hvd.DistributedOptimizer(base, named_parameters=model.named_parameters())
        hvd.broadcast_parameters(model.state_dict(), root_rank=0)
        eng = opt.fused_engine
        our_launches = lambda: (eng.kernel_launches if eng is not None else 0) + counters.total()
        step_model = model
    else:
        opt = base
        if world > 1:
            step_model = torch.nn.parallel.DistributedDataParallel(
                model, device_ids=[dev.index], gradient_as_bucket_view=True)
        else:
            step_model = model

    data = wl.data()
    dev_batches = [data.next() for _ in range(2)]      # device-resident inputs for the device-timed region
    torch.cuda.synchronize()

    def eager_step(x, y):
        loss = wl.loss(step_model(x), y)
        loss.backward()
        opt.step()
        opt.zero_grad(set_to_none=(impl != "ours"))
        return loss.detach()

    train_step, graphed, gs = eager_step, False, None
    if impl == "ours" and graph_mode != "off" and eng is not None:
        from distributed_torch_horovod_gcp_b200.utils.graph import GraphedStep
        ok = True
        try:
            gs = GraphedStep(eager_step, list(dev_batches[0]), warmup=3)
        except Exception as e:  # noqa: BLE001
            ok = False
            if graph_mode == "on":
                raise
            print(f"[bench] CUDA-graph capture failed ({type(e).__name__}: {e}); running eager",
                  file=sys.stderr)
        if world > 1:      # all ranks must take the same path (graphs replay collectives)
            ok = all(hvd.allgather_object(ok))
        if ok:
            train_step, graphed = gs, True

    def sync_all():
        torch.cuda.synchronize()
        if world > 1:
            hvd.barrier()
        torch.cuda.synchronize()

    def max_over_ranks(v: float) -> float:
        if world == 1:
            return v
        t = torch.tensor([v], dtype=torch.float64)
        return float(hvd.allreduce(t, op=hvd.Max))

    for i in range(max(warmup, 3)):
        loss = train_step(*dev_batches[i % 2])
    float(loss)
    sync_all()

    sampler = ClockSampler(dev.index).start() if (rank == 0 and want_clocks) else None
    l0 = our_launches()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    sync_all()
    e0.record()
    for i in range(steps):
        loss = train_step(*dev_batches[i % 2])
    e1.record()
    sync_all()
    ms = max_over_ranks(e0.elapsed_time(e1))
    launches = our_launches() - l0
    if graphed:
        launches = gs.kernels_per_replay * steps          # replayed graph nodes, counted at capture
    final_loss = float(loss)
    if dump_dir is not None and rank == 0:
        dump_outputs(dump_dir, loss, model)

    e2e = None
    if want_e2e:
        host_loss = torch.zeros(steps, dtype=torch.float32).pin_memory()
        evs = []
        for i in range(3):
            train_step(*data.next())
        sync_all()
        e0.record()
        for i in range(steps):
            x, y = data.next()                       # H2D of this step's inputs (pinned -> device)
            loss = train_step(x, y)
            host_loss[i:i + 1].copy_(loss.detach().reshape(1), non_blocking=True)   # D2H result
            ev = torch.cuda.Event()
            ev.record()
            evs.append(ev)
            if i >= 1:
                evs[i - 1].synchronize()             # the training loop consumes the previous loss
                _ = float(host_loss[i - 1])
        e1.record()
        sync_all()
        ms_e2e = max_over_ranks(e0.elapsed_time(e1))
        e2e = {"value": round(wl.batch * world * steps / (ms_e2e / 1e3), 2),
               "unit": "samples/sec", "ms_per_step": round(ms_e2e / steps, 4),
               "h2d_bytes_per_step": int(data.bytes_per_batch), "d2h_bytes_per_step": 4}
    clocks = sampler.stop() if sampler is not None else None
    comm = "none"
    if impl == "ours":
        comm = eng.algorithms() if eng is not None else (
            "none" if world == 1 else "NCCL FALLBACK (symmetric runtime unavailable): bucketed "
            "allreduce + torch optimizer")
    elif world > 1:
        comm = "nccl-ddp"
    res = {"ms": ms, "value": wl.batch * world * steps / (ms / 1e3), "launches": int(launches),
           "final_loss": final_loss, "graphed": graphed, "e2e": e2e, "clocks": clocks, "comm": comm,
           "model": model, "opt": opt}
    F2._FORCE_REFERENCE = False
    return res


def selfcheck(wl, hvd, world, rank):
    """Reduction + update check at N > 1, with IDENTICAL local gradients on both arms: one backward on
    a plain clone produces per-rank gradients; (a) ``dist.all_reduce`` (NCCL) average + the stock torch
    optimizer update the clone, (b) the same local gradients are placed in the fused engine's gradient
    buckets and ONE fused sm_90a launch per bucket reduces them over NVLink and updates the model.
    Also checks that the updated replicas are bit-identical across ranks."""
    import copy
    import hashlib
    import torch
    import torch.distributed as dist
    os.environ.setdefault("B200DP_FUSED_SINGLE", "1")
    model = wl.build_model(seed=99)
    opt = hvd.DistributedOptimizer(wl.build_optimizer(model), named_parameters=model.named_parameters())
    hvd.broadcast_parameters(model.state_dict(), root_rank=0)
    ref = copy.deepcopy(model)
    for p in ref.parameters():
        p.grad = None
        if hasattr(p, "_b200dp_sink"):
            del p._b200dp_sink
    ropt = wl.build_optimizer(ref)
    x, y = wl.data().next()
    wl.loss(ref(x), y).backward()                      # local gradients (plain autograd accumulation)
    with torch.no_grad():
        for p, q in zip(model.parameters(), ref.parameters()):
            p.grad.copy_(q.grad)                       # same bits into the fused engine's buckets
    opt.step()                                         # synchronize(): every bucket launched once
    opt.zero_grad()
    for p in ref.parameters():
        g = p.grad.float()
        dist.all_reduce(g)
        p.grad.copy_((g / world).to(p.grad.dtype))
    ropt.step()
    torch.cuda.synchronize()
    worst = 0.0
    for p, q in zip(model.parameters(), ref.parameters()):
        a, b = p.detach().float(), q.detach().float()
        worst = max(worst, float((a - b).abs().max() / b.abs().max().clamp_min(1e-12)))
    h = hashlib.sha256()
    for p in model.parameters():
        h.update(p.detach().contiguous().view(torch.uint8).cpu().numpy().tobytes())
    digests = hvd.allgather_object(h.hexdigest())
    opt.remove_hooks()
    return {"max_rel_err": worst, "replicas_bit_identical": len(set(digests)) == 1,
            "expected": ("a few bf16 ulps (2^-8 = 0.0039 each): the NCCL arm rounds the reduced gradient to bf16 "
                         "and torch updates bf16 parameters in bf16; the fused engine sums in fp32 (another "
                         "order) and rounds the fp32 master once"
                         if wl.dtype_name == "bf16" else "fp32 rounding (~1e-6)"),
            "what": "fused NVLink allreduce+update vs NCCL all_reduce + torch optimizer on identical "
                    "local gradients; per-tensor max|a-b| / max|b|, worst tensor"}


def main():
    args = parse()
    if args.impl == "reference":
        return reference_arm(args)
    import torch
    import distributed_torch_horovod_gcp_b200.torch as hvd

    if not torch.cuda.is_available():
        print(json.dumps({"error": "bench.py needs a CUDA device", "n_gpus": 0}), flush=True)
        return 1
    hvd.init()
    rank, world = hvd.rank(), hvd.size()
    if world != args.gpus and rank == 0:
        print(f"[bench] warning: --gpus {args.gpus} but world size is {world}", file=sys.stderr)
    torch.cuda.set_device(hvd.local_rank())
    dev = torch.device("cuda", torch.cuda.current_device())
    torch.backends.cudnn.benchmark = True
    wl = Workload(args, dev, rank)

    main_res = run_arm(args.impl, wl, hvd, world, rank, args.steps, args.warmup, args.graph,
                       want_e2e=not args.no_e2e, want_clocks=True, dump_dir=args.dump_outputs)
    main_res.pop("model")
    opt = main_res.pop("opt")
    if hasattr(opt, "remove_hooks"):
        opt.remove_hooks()
    del opt
    torch.cuda.empty_cache()

    base_res = None
    if args.impl == "ours" and not args.no_baseline:
        try:
            base_res = run_arm("nccl_standin", wl, hvd, world, rank, min(args.steps, 10), 3, "off",
                               want_e2e=False, want_clocks=False)
            base_res.pop("model")
            base_res.pop("opt")
            torch.cuda.empty_cache()
        except Exception as e:  # noqa: BLE001
            print(f"[bench] stand-in arm failed: {type(e).__name__}: {e}", file=sys.stderr)
            base_res = None
    check = None
    if args.impl == "ours" and world > 1 and not args.no_selfcheck:
        try:
            check = selfcheck(wl, hvd, world, rank)
        except Exception as e:  # noqa: BLE001
            check = {"error": f"{type(e).__name__}: {e}"}

    if rank == 0:
        unit = "samples/sec" if wl.is_lstm else "images/sec"
        metric = ("images/sec (whole job, device-timed, max over ranks) ResNet-50 synthetic ImageNet "
                  "training" if args.model == "resnet50" else
                  f"{unit} (whole job, device-timed, max over ranks) {args.model} training")
        e2e = main_res["e2e"]
        if e2e is not None:
            e2e["unit"] = unit
        line = {
            "metric": metric, "value": round(main_res["value"], 2), "unit": unit, "n_gpus": world,
            "steps": args.steps, "warmup": max(args.warmup, 3),
            "ms_per_step": round(main_res["ms"] / args.steps, 4),
            "higher_is_better": True, "scaling": "weak",
            "vs_baseline": (round(main_res["value"] / base_res["value"], 3) if base_res else None),
            "baseline_kind": ("NCCL stand-in measured in this run (same model on cuDNN/cuBLAS ops + NCCL DDP + "
                              "torch optimizer, eager) — NOT Horovod, NOT the reference (uninstallable "
                              "offline, DESIGN.md §0); BASELINE.md has no published number"
                              if base_res else None),
            "baseline": ({"value": round(base_res["value"], 2),
                          "ms_per_step": round(base_res["ms"] / min(args.steps, 10), 4),
                          "steps": min(args.steps, 10), "comm": base_res["comm"]} if base_res else None),
            "dtype": wl.dtype_name,
            "data": "synthetic (random inputs/labels of the benchmark's shape, random-init weights)",
            "impl": args.impl,
            "config": {"model": args.model, "global_batch": wl.batch * world,
                       "per_gpu_batch": wl.batch,
                       **({"seq_len": 10, "features": 23, "hidden": 256} if wl.is_lstm else
                          {"image_size": args.image_size, "layout": "NHWC bf16"}),
                       "parallelism": f"dp{world}", "optimizer": wl.optimizer_name(),
                       "cuda_graph": main_res["graphed"],
                       "l2": ("launch/latency-bound config: working set (2 MB) lives in L2 by design"
                              if wl.is_lstm else
                              "no explicit flush: per-step working set (activations, several GB) >> 50 MB L2"),
                       "comm": main_res["comm"]},
            "clocks": main_res["clocks"], "e2e": e2e,
            "gpu_launches": main_res["launches"],
            "gpu_launches_note": "hand-written sm_90a kernels of this repo inside the timed region "
                                 "(ATen glue such as loss / pooling kernels is not counted)",
            "selfcheck": check,
            "final_loss": round(main_res["final_loss"], 6),
        }
        print(json.dumps(line), flush=True)
    hvd.shutdown()
    return 0


if __name__ == "__main__":
    sys.exit(main())
