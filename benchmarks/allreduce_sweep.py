#!/usr/bin/env python
"""Gradient all-reduce bandwidth sweep, 1 KB – 1 GB ([DRIVER] BASELINE.json config 5):
the framework's sm_90a kernels (one-shot / two-shot / NVLS, and the auto choice) against
``torch.distributed`` NCCL on the same buffers.

    python -m torch.distributed.run --nproc-per-node 8 --master-addr 127.0.0.1 --master-port 29533 \
        benchmarks/allreduce_sweep.py --out allreduce_sweep_8.json

Every number is device-timed (CUDA events around ``iters`` back-to-back collectives on the
launching stream, barrier + synchronize on both sides) and is the MAX over ranks.
bus GB/s = 2 (N-1)/N * bytes / t   (NCCL-tests convention); roofline = NVLink per-direction
bandwidth (H100 SXM, NVLink 4: 450 GB/s nominal).
Buffers live in symmetric memory (zero-copy, in place), like NCCL's in-place all-reduce.
Small sizes are L2-resident by nature (latency regime); sizes >= 256 MB exceed the 50 MB L2.
"""
import argparse
import json
import os
import sys

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import distributed_torch_horovod_gcp_b200.torch as hvd  # noqa: E402
from distributed_torch_horovod_gcp_b200 import _state  # noqa: E402
from distributed_torch_horovod_gcp_b200.runtime import symm as S  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--min-bytes", type=int, default=1 << 10)
    ap.add_argument("--max-bytes", type=int, default=1 << 30)
    ap.add_argument("--dtype", default="fp32", choices=["fp32", "bf16"])
    ap.add_argument("--out", default="")
    ap.add_argument("--algos", default="auto,oneshot,twoshot,nvls,nccl")
    ap.add_argument("--write-tuning", default="",
                    help="derive the algorithm table for this world size from the sweep and write "
                         "it as JSON (load with B200DP_TUNING_FILE)")
    args = ap.parse_args()

    hvd.init()
    rank, world = hvd.rank(), hvd.size()
    torch.cuda.set_device(hvd.local_rank())
    dev = torch.device("cuda", torch.cuda.current_device())
    symm = _state.get_symm()
    assert symm is not None, f"symmetric runtime unavailable: {_state.runtime().symm_failed}"
    dtype = torch.float32 if args.dtype == "fp32" else torch.bfloat16
    es = 4 if dtype == torch.float32 else 2
    buf = symm.alloc(args.max_bytes)
    full = buf.tensor(dtype)
    full.fill_(1.0)
    nccl_buf = torch.ones(args.max_bytes // es, dtype=dtype, device=dev)
    algos = [a for a in args.algos.split(",") if a]
    code = {"oneshot": S.ALGO_ONESHOT, "twoshot": S.ALGO_TWOSHOT, "nvls": S.ALGO_NVLS}

    def timed(fn, iters, warm):
        for _ in range(warm):
            fn()
        torch.cuda.synchronize()
        hvd.barrier()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(iters):
            fn()
        e1.record()
        torch.cuda.synchronize()
        hvd.barrier()
        ms = e0.elapsed_time(e1) / iters
        t = torch.tensor([ms], dtype=torch.float64)
        return float(hvd.allreduce(t, op=hvd.Max))

    rows = []
    nbytes = args.min_bytes
    while nbytes <= args.max_bytes:
        n = nbytes // es
        view = full[:n]
        iters = 200 if nbytes <= (1 << 20) else (40 if nbytes <= (64 << 20) else 10)
        warm = 10 if nbytes <= (1 << 20) else 3
        row = {"bytes": nbytes}
        for a in algos:
            if a == "nccl":
                nv = nccl_buf[:n]
                ms = timed(lambda: dist.all_reduce(nv), iters, warm)
            elif a == "auto":
                fn = symm.prepare_allreduce(view, 1.0 / world)
                ms = timed(fn, iters, warm)
                row["auto_algo"] = fn.algo
            else:
                if a == "nvls" and not (symm.multicast and buf.mc_ptr):
                    continue
                if a == "oneshot" and nbytes > (64 << 20):
                    continue                      # (N-1)x traffic: pointless and slow at these sizes
                fn = symm.prepare_allreduce(view, 1.0 / world, algo=code[a])
                ms = timed(fn, iters, warm)
            row[a + "_us"] = round(ms * 1e3, 2)
            row[a + "_busGBs"] = round(2 * (world - 1) / world * nbytes / (ms * 1e-3) / 1e9, 2)
            full.fill_(1.0)
        symm.check_errors()
        rows.append(row)
        if rank == 0:
            print(json.dumps(row), flush=True)
        nbytes *= 4
    if rank == 0 and args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump({"world": world, "dtype": args.dtype, "multicast": bool(symm.multicast),
                       "roofline_GBs": {"nvlink_nominal_per_dir_h100_sxm_datasheet": 450},
                       "rows": rows}, f, indent=1)
    if rank == 0 and args.write_tuning:
        from distributed_torch_horovod_gcp_b200.runtime import tuning
        tab = {}
        if os.path.exists(args.write_tuning):
            with open(args.write_tuning) as f:
                tab = json.load(f)
        tab[str(world)] = tuning.derive_from_sweep(rows, world, bool(symm.multicast))
        with open(args.write_tuning, "w") as f:
            json.dump(tab, f, indent=1)
    hvd.shutdown()


if __name__ == "__main__":
    main()
