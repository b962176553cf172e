"""Algorithm-selection table for the comm kernels — the replacement for Horovod's autotuner
(`HOROVOD_AUTOTUNE` / parameter_manager: Bayesian search over fusion threshold and cycle time;
SURVEY.md §2.2 N11, §5.6).  There is nothing to search at run time here: the bucket plan is
static and the only choice is WHICH kernel reduces a bucket of a given size on a given world
size.  The default table below is a starting point, not a measurement of any particular machine;
`benchmarks/allreduce_sweep.py --write-tuning FILE` derives one for the machine it runs on and
`B200DP_TUNING_FILE=FILE` makes every rank load it.

Table format (JSON): {"<world>": {"oneshot_max_bytes": int, "prefer": "nvls" | "twoshot"}, ...}
"""
from __future__ import annotations

import json
import os
from typing import Dict, Optional

ONESHOT, TWOSHOT, NVLS = 0, 1, 2

DEFAULT_TABLE: Dict[str, dict] = {
    "2": {"oneshot_max_bytes": 8 << 10, "prefer": "twoshot"},
    "default": {"oneshot_max_bytes": 8 << 10, "prefer": "nvls"},
}

_loaded: Optional[Dict[str, dict]] = None


def table() -> Dict[str, dict]:
    global _loaded
    if _loaded is None:
        _loaded = dict(DEFAULT_TABLE)
        path = os.environ.get("B200DP_TUNING_FILE")
        if path and os.path.exists(path):
            with open(path) as f:
                user = json.load(f)
            for k, v in user.items():
                if isinstance(v, dict) and "oneshot_max_bytes" in v:
                    _loaded[str(k)] = {"oneshot_max_bytes": int(v["oneshot_max_bytes"]),
                                       "prefer": str(v.get("prefer", "nvls"))}
    return _loaded


def reset() -> None:
    global _loaded
    _loaded = None


def choose(world: int, nbytes: int, multicast: bool) -> int:
    """Pure function: algorithm for a bucket of ``nbytes`` on ``world`` ranks."""
    t = table()
    row = t.get(str(world), t["default"])
    if nbytes <= row["oneshot_max_bytes"]:
        return ONESHOT
    if row["prefer"] == "nvls" and multicast and world > 2:
        return NVLS
    return TWOSHOT


def derive_from_sweep(rows, world: int, multicast: bool) -> dict:
    """Turn allreduce_sweep rows ({bytes, oneshot_us, twoshot_us, nvls_us}) into a table row: the
    largest size at which one-shot is still the fastest kernel, and the better sliced kernel at
    the largest measured size."""
    oneshot_max = 0
    for r in sorted(rows, key=lambda r: r["bytes"]):
        cands = {k: r[k + "_us"] for k in ("oneshot", "twoshot", "nvls") if k + "_us" in r}
        if not cands:
            continue
        if min(cands, key=cands.get) == "oneshot":
            oneshot_max = r["bytes"]
        else:
            break
    last = max(rows, key=lambda r: r["bytes"])
    prefer = "twoshot"
    if multicast and "nvls_us" in last and last["nvls_us"] <= last.get("twoshot_us", float("inf")):
        prefer = "nvls"
    return {"oneshot_max_bytes": int(oneshot_max), "prefer": prefer}


def autotune(symm, sizes=(4 << 10, 16 << 10, 64 << 10, 256 << 10, 1 << 20, 4 << 20, 16 << 20),
             iters: int = 8) -> dict:
    """``horovodrun --autotune`` / ``HOROVOD_AUTOTUNE=1``: measure the three allreduce kernels on THIS
    machine at start-up (collective; ~0.2 s) and install the derived row for this world size — the
    measured replacement for Horovod's Bayesian parameter_manager.  Times are CUDA-event device times,
    max over ranks."""
    import torch
    import torch.distributed as dist
    global _loaded
    world = symm.world
    buf = symm.alloc_tensor(max(sizes) // 4, torch.float32)
    buf.zero_()
    rows = []
    algos = [("oneshot", ONESHOT), ("twoshot", TWOSHOT)] + ([("nvls", NVLS)] if symm.multicast else [])
    for nbytes in sizes:
        t = buf[: nbytes // 4]
        row = {"bytes": nbytes}
        for name, code in algos:
            launch = symm.prepare_allreduce(t, scale=1.0, algo=code)
            for _ in range(2):
                launch()
            torch.cuda.synchronize(symm.device)
            dist.barrier(group=symm.group)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(iters):
                launch()
            e1.record()
            torch.cuda.synchronize(symm.device)
            us = torch.tensor([e0.elapsed_time(e1) * 1e3 / iters], dtype=torch.float64)
            dist.all_reduce(us, op=dist.ReduceOp.MAX, group=symm.group)
            row[name + "_us"] = float(us)
        rows.append(row)
    derived = derive_from_sweep(rows, world, bool(symm.multicast))
    table()[str(world)] = derived
    symm.check_errors()
    return {"rows": rows, "table": derived}
