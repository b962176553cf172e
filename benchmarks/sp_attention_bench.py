#!/usr/bin/env python
"""Sequence-parallel causal flash attention (csrc/attn_sm90.cu, ops/seq_parallel.py): per-rank kernel times at
world sizes 1, 2, 4 and 8, emulated on one GPU.

Configuration: causal, B = 1, H = 12 (B·H = 12), head dim 64, S in {8192, 16384, 32768} (the global sequence).
For each (S, W) every emulated rank r runs ``b200dp_attn_sp_fwd`` and ``b200dp_attn_sp_bwd`` on its zigzag shard
against gathered operands built on this GPU (the kernels read other ranks' data only through those buffers, so
this is the work rank r's GPU does).  Printed per (S, W): each rank's forward and backward kernel time, the
max / min ratio over ranks (the balance the zigzag sharding is for), and the sum over ranks against one
full-sequence kernel (``b200dp_attn_fwd_ex`` / ``b200dp_attn_bwd``; the latter includes its delta pass, which
the sequence-parallel op runs in its backward pack, timed per rank as ``rank_pack_bwd_ms``: the Q|dO|LSE copies
and ``b200dp_attn_delta``).
With 2 or more GPUs it also times the real op (``sp_attention`` forward + backward, collectives included) at
each world size that fits.  CUDA events, --warmup untimed calls, median of --iters; the card name and power limit
are read in the same run and printed with the numbers."""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True)
    name, power = [s.strip() for s in q.stdout.splitlines()[0].split(",")]
    return name, power


def timeit(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    ts.sort()
    return ts[len(ts) // 2]


def full_kernels(q, k, v, do, iters, warmup):
    """Times (ms) of one full-sequence causal forward and backward."""
    from distributed_torch_horovod_gcp_b200.ops import attention as A
    B, H, S, D = q.shape
    st = torch.cuda.current_stream().cuda_stream
    o = torch.empty((B, S, H, D), dtype=torch.bfloat16, device="cuda").permute(0, 2, 1, 3)
    lse = torch.empty((B, H, S), dtype=torch.float32, device="cuda")
    delta = torch.empty_like(lse)
    acc = torch.zeros((B, S, H, D), dtype=torch.float32, device="cuda")
    acc_v = acc.permute(0, 2, 1, 3)
    dk, dv = torch.empty_like(o), torch.empty_like(o)
    s = A._strides

    def fwd():
        A._ck(A._lib.b200dp_attn_fwd_ex(q.data_ptr(), k.data_ptr(), v.data_ptr(), o.data_ptr(), lse.data_ptr(), B, H,
                                        S, D, s(q), s(k), s(v), s(o), 0.125, 1, st))

    def bwd():
        A._ck(A._lib.b200dp_attn_bwd(q.data_ptr(), k.data_ptr(), v.data_ptr(), o.data_ptr(), do.data_ptr(),
                                     lse.data_ptr(), delta.data_ptr(), acc.data_ptr(), dk.data_ptr(), dv.data_ptr(), B,
                                     H, S, D, s(q), s(k), s(v), s(o), s(do), s(acc_v), s(dk), s(dv), 0.125, 1, st))
    t_f = timeit(fwd, iters, warmup)
    t_b = timeit(bwd, iters, warmup)
    return t_f, t_b, o, lse


def emulated(q, k, v, do, o, lse, W, iters, warmup):
    """Per-rank times (ms) of the sequence-parallel forward and backward kernels, and of the backward pack
    (Q|dO|LSE copies and the delta kernel), at world size W."""
    from distributed_torch_horovod_gcp_b200.ops import seq_parallel as sp
    B, H, S, D = q.shape
    S_loc = S // W
    sh = (lambda t, r: sp.zigzag_shard(t, 2, r, W))
    loc = [[sh(t, r) for t in (q, k, v, do, o, lse)] for r in range(W)]
    kg, vg = sp.kv_views(torch.stack([sp.pack_kv(l[1], l[2]) for l in loc]))
    g = torch.stack([sp.pack_bwd(l[0], l[3], l[4], l[5]) for l in loc])
    qg, dog, lse_ptr, delta_ptr, ld_sw = sp.bwd_views(g, B, H, S_loc)
    acc = torch.zeros((W, B, S_loc, H, D), dtype=torch.float32, device="cuda").permute(0, 1, 3, 2, 4)
    rows = []
    for r in range(W):
        lq, lk, lv, ldo, lo, llse = loc[r]
        o_r = torch.empty_like(lo)
        lse_r = torch.empty_like(llse)
        dk, dv = torch.empty_like(lk), torch.empty_like(lv)
        t_f = timeit(lambda: sp.sp_fwd(lq, kg, vg, o_r, lse_r, True, r, W), iters, warmup)
        t_b = timeit(lambda: sp.sp_bwd(qg, lk, lv, dog, lse_ptr, delta_ptr, ld_sw, acc, dk, dv, True, r, W),
                     iters, warmup)
        t_d = timeit(lambda: sp.pack_bwd(lq, ldo, lo, llse), iters, warmup)
        rows.append((t_f, t_b, t_d))
    return rows


# ------------------------------------------------------------------ real op on W GPUs
def _real_worker(rank, world, port, S, iters, warmup, q_out):
    os.environ.update({"RANK": str(rank), "WORLD_SIZE": str(world), "LOCAL_RANK": str(rank),
                       "LOCAL_WORLD_SIZE": str(world), "MASTER_ADDR": "127.0.0.1", "MASTER_PORT": str(port)})
    torch.cuda.set_device(rank)
    import distributed_torch_horovod_gcp_b200.torch as hvd
    from distributed_torch_horovod_gcp_b200.ops import seq_parallel as sp
    hvd.init()
    try:
        S_loc = S // world
        g = torch.Generator(device="cuda").manual_seed(rank)
        mats = [torch.randn(S_loc, 12 * 64, generator=g, device="cuda").bfloat16().requires_grad_(True)
                for _ in range(3)]
        q, k, v = [m.view(1, S_loc, 12, 64).transpose(1, 2) for m in mats]
        do = torch.randn(1, S_loc, 12, 64, generator=g, device="cuda").bfloat16().transpose(1, 2)

        def step():
            sp.sp_attention(q, k, v, causal=True).backward(do)
        t = timeit(step, iters, warmup)
        ts = hvd.allgather(torch.tensor([t], dtype=torch.float64))
        if rank == 0:
            q_out.put(ts.tolist())
    finally:
        hvd.shutdown()


def real_op(world, S, iters, warmup):
    import socket
    import torch.multiprocessing as mp
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_real_worker, args=(r, world, port, S, iters, warmup, q)) for r in range(world)]
    for p in procs:
        p.start()
    try:
        return q.get(timeout=600)
    finally:
        for p in procs:
            p.join(timeout=60)


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawTextHelpFormatter)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--seqs", default="8192,16384,32768")
    ap.add_argument("--worlds", default="1,2,4,8")
    ap.add_argument("--out", default=None, help="also write the rows to this JSON file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("sp_attention_bench needs a GPU")
    from distributed_torch_horovod_gcp_b200.ops import kernels
    assert kernels.has("attention_fused"), "attention kernels missing"
    name, power = card()
    B, H = 1, 12
    rows = []
    for S in [int(x) for x in args.seqs.split(",")]:
        g = torch.Generator().manual_seed(S)
        q, k, v, do = [torch.randn(B, H, S, 64, generator=g).bfloat16().cuda() for _ in range(4)]
        t_ff, t_fb, o, lse = full_kernels(q, k, v, do, args.iters, args.warmup)
        for W in [int(x) for x in args.worlds.split(",")]:
            per = emulated(q, k, v, do, o, lse, W, args.iters, args.warmup)
            f, b, d = [[p[i] for p in per] for i in range(3)]
            row = {"gpu": name, "power_limit": power, "S": S, "W": W, "B": B, "H": H, "d": 64, "causal": True,
                   "rank_fwd_ms": [round(x, 4) for x in f], "rank_bwd_ms": [round(x, 4) for x in b],
                   "rank_pack_bwd_ms": [round(x, 4) for x in d],
                   "fwd_max_over_min": round(max(f) / min(f), 3), "bwd_max_over_min": round(max(b) / min(b), 3),
                   "fwd_sum_ms": round(sum(f), 3), "bwd_sum_ms": round(sum(b), 3),
                   "full_fwd_ms": round(t_ff, 3), "full_bwd_ms": round(t_fb, 3),
                   "fwd_sum_over_full": round(sum(f) / t_ff, 3), "bwd_sum_over_full": round(sum(b) / t_fb, 3)}
            rows.append(row)
            print(json.dumps(row), flush=True)
        del q, k, v, do, o, lse
        torch.cuda.empty_cache()
    ngpu = torch.cuda.device_count()
    for W in [int(x) for x in args.worlds.split(",")]:
        if 2 <= W <= ngpu:
            for S in [int(x) for x in args.seqs.split(",")]:
                ts = real_op(W, S, args.iters, args.warmup)
                row = {"gpu": name, "power_limit": power, "S": S, "W": W, "real_op_fwd_bwd_ms_per_rank":
                       [round(t, 3) for t in ts]}
                rows.append(row)
                print(json.dumps(row), flush=True)
    if ngpu < 2:
        print(json.dumps({"real_op": "not measured: one GPU"}), flush=True)
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as fh:
            json.dump(rows, fh, indent=1)


if __name__ == "__main__":
    main()
