"""Process-wide runtime state: rank/size/topology, control-plane process group, backends.

Replaces Horovod's C++ global state + controller (SURVEY.md §2.2 N1/N2; reached from
reference app/torch_train.py:210,217,227,232).  Design differences, H100-first:

* No background polling thread and no per-tensor negotiation: the data-parallel bucket
  plan is static and identical on all ranks, so ordering is by bucket index and
  completion is CUDA-stream ordered (events), never host polled.
* The control plane (rendezvous, handle exchange, plan-hash check) is a Gloo CPU group
  from ``torch.distributed``; it is used at init / setup time only.
* The data plane for CUDA tensors is the symmetric-memory runtime in
  ``runtime/`` (cuMem VMM peer mappings + NVLS multicast) driven by the sm_90a
  kernels in ``csrc/comm_kernels.cu``.  NCCL is only a loud fallback.
"""
from __future__ import annotations

import datetime
import logging
import os
import threading
from dataclasses import dataclass, field
from typing import Optional

import torch
import torch.distributed as dist

log = logging.getLogger("b200dp")


def _env_int(*names: str, default: Optional[int] = None) -> Optional[int]:
    for n in names:
        v = os.environ.get(n)
        if v is not None and v != "":
            try:
                return int(v)
            except ValueError:
                pass
    return default


def launch_size() -> int:
    """The world size the launcher's environment gives (1 without a launcher): what ``init`` will use."""
    return _env_int("HOROVOD_SIZE", "WORLD_SIZE", "OMPI_COMM_WORLD_SIZE", "PMI_SIZE", default=1)


@dataclass
class Runtime:
    initialized: bool = False
    rank: int = 0
    size: int = 1
    local_rank: int = 0
    local_size: int = 1
    cross_rank: int = 0
    cross_size: int = 1
    owns_pg: bool = False
    cpu_group: Optional[object] = None      # gloo group for control plane + CPU tensors
    symm: Optional[object] = None           # runtime.symm.SymmRuntime (lazy, CUDA only)
    symm_failed: Optional[str] = None       # reason string if symmetric runtime setup failed
    timeline: Optional[object] = None
    lock: threading.RLock = field(default_factory=threading.RLock)
    process_sets: dict = field(default_factory=dict)


_RT = Runtime()


def runtime() -> Runtime:
    return _RT


def _require_init() -> Runtime:
    if not _RT.initialized:
        raise ValueError(
            "distributed_torch_horovod_gcp_b200 has not been initialized; use hvd.init().")
    return _RT


def init(comm=None, process_sets=None) -> None:
    """Idempotent initialisation (Horovod ``hvd.init()`` semantics, reference
    app/torch_train.py:210).

    Reads the launcher environment (our launcher / torchrun: ``RANK``, ``WORLD_SIZE``,
    ``LOCAL_RANK``, ``LOCAL_WORLD_SIZE``; Horovod-compatible: ``HOROVOD_RANK`` …;
    OpenMPI: ``OMPI_COMM_WORLD_*``).  With no launcher it becomes rank 0 / size 1 — the
    single-GPU path of the reference README (README.md:20-23).  Does not select a CUDA
    device; the caller pins the device afterwards (app/torch_train.py:232).
    """
    rt = _RT
    with rt.lock:
        if rt.initialized:
            return
        rank = _env_int("HOROVOD_RANK", "RANK", "OMPI_COMM_WORLD_RANK", "PMI_RANK", default=0)
        size = launch_size()
        local_rank = _env_int("HOROVOD_LOCAL_RANK", "LOCAL_RANK",
                              "OMPI_COMM_WORLD_LOCAL_RANK", default=None)
        local_size = _env_int("HOROVOD_LOCAL_SIZE", "LOCAL_WORLD_SIZE",
                              "OMPI_COMM_WORLD_LOCAL_SIZE", default=None)
        if local_size is None:
            local_size = size
        if local_rank is None:
            local_rank = rank % max(local_size, 1)
        cross_size = _env_int("HOROVOD_CROSS_SIZE", default=max(size // max(local_size, 1), 1))
        cross_rank = _env_int("HOROVOD_CROSS_RANK", default=rank // max(local_size, 1))

        if dist.is_available() and dist.is_initialized():
            # Adopt an existing process group (e.g. created by the user / torchrun script).
            rank, size = dist.get_rank(), dist.get_world_size()
            rt.owns_pg = False
        elif size > 1:
            os.environ.setdefault("MASTER_ADDR", os.environ.get(
                "HOROVOD_GLOO_RENDEZVOUS_ADDR", "127.0.0.1"))
            os.environ.setdefault("MASTER_PORT", os.environ.get(
                "HOROVOD_GLOO_RENDEZVOUS_PORT", "29500"))
            timeout_s = _env_int("HOROVOD_START_TIMEOUT", "B200DP_START_TIMEOUT", default=600)
            use_cuda = torch.cuda.is_available() and os.environ.get("B200DP_FORCE_CPU", "0") != "1"
            backend = "cpu:gloo,cuda:nccl" if use_cuda else "gloo"
            dist.init_process_group(
                backend=backend, rank=rank, world_size=size,
                timeout=datetime.timedelta(seconds=timeout_s))
            rt.owns_pg = True

        rt.rank, rt.size = rank, size
        rt.local_rank, rt.local_size = local_rank, local_size
        rt.cross_rank, rt.cross_size = cross_rank, cross_size
        if size > 1:
            # Dedicated Gloo group: control plane + CPU-tensor collectives.
            try:
                rt.cpu_group = dist.new_group(backend="gloo")
            except Exception:
                rt.cpu_group = dist.group.WORLD
        rt.initialized = True
        lvl = os.environ.get("HOROVOD_LOG_LEVEL") or os.environ.get("B200DP_LOG_LEVEL")
        if lvl:      # horovodrun --log-level: TRACE/DEBUG/INFO/WARNING/ERROR/FATAL -> the package logger
            lv = {"TRACE": logging.DEBUG, "FATAL": logging.CRITICAL}.get(lvl.upper(),
                                                                         getattr(logging, lvl.upper(), None))
            if lv is not None:
                log.setLevel(lv)
                if not log.handlers:
                    h = logging.StreamHandler()
                    h.setFormatter(logging.Formatter(f"[b200dp rank {rank}] %(levelname)s %(message)s"))
                    log.addHandler(h)
        log.debug("init: rank %d/%d local %d/%d", rank, size, local_rank, local_size)
        tl = os.environ.get("HOROVOD_TIMELINE") or os.environ.get("B200DP_TIMELINE")
        if tl:
            from .utils.timeline import Timeline
            rt.timeline = Timeline(tl, rank)


def shutdown() -> None:
    rt = _RT
    with rt.lock:
        if not rt.initialized:
            return
        if rt.timeline is not None:
            try:
                rt.timeline.close()
            finally:
                rt.timeline = None
        try:      # engines hold views of symmetric arenas: detach the models before unmapping
            from .parallel.fused_engine import live_engines
            for eng in live_engines():
                eng.release()
        except Exception:
            pass
        if rt.symm is not None:
            try:
                rt.symm.close()
            except Exception:
                pass
            rt.symm = None
            # physical memory of a symmetric allocation is returned when the LAST handle to it goes — the
            # peers' imported handles included: wait until every rank has closed before reporting done
            try:
                if rt.cpu_group is not None and dist.is_initialized() and rt.size > 1:
                    import datetime
                    dist.monitored_barrier(group=rt.cpu_group, timeout=datetime.timedelta(seconds=10))
            except Exception:      # a dead peer must not block teardown
                pass
        if rt.owns_pg and dist.is_initialized():
            try:
                dist.destroy_process_group()
            except Exception:
                pass
        rt.cpu_group = None
        rt.initialized = False
        rt.rank, rt.size, rt.local_rank, rt.local_size = 0, 1, 0, 1
        rt.cross_rank, rt.cross_size = 0, 1
        rt.owns_pg = False
        rt.symm_failed = None
        rt.process_sets.clear()


def is_initialized() -> bool:
    return _RT.initialized


def rank() -> int:
    return _require_init().rank


def size() -> int:
    return _require_init().size


def local_rank() -> int:
    return _require_init().local_rank


def local_size() -> int:
    return _require_init().local_size


def cross_rank() -> int:
    return _require_init().cross_rank


def cross_size() -> int:
    return _require_init().cross_size


def is_homogeneous() -> bool:
    rt = _require_init()
    return rt.size % max(rt.local_size, 1) == 0


def get_symm(device: Optional[torch.device] = None):
    """Return the symmetric-memory runtime for the current CUDA device, creating it on
    first use (collective call: every rank must reach this).  Returns ``None`` if the
    runtime is unavailable (no CUDA, world size 1, multi-host, or setup failure — the
    reason is kept in ``runtime().symm_failed`` and reported loudly once)."""
    rt = _require_init()
    if rt.symm is not None:
        return rt.symm
    if rt.symm_failed is not None or rt.size == 1 or not torch.cuda.is_available():
        return None
    if os.environ.get("B200DP_DISABLE_SYMM", "0") == "1":
        rt.symm_failed = "disabled by B200DP_DISABLE_SYMM=1"
        return None
    from .runtime.symm import SymmRuntime
    err = None
    try:
        symm = SymmRuntime.create(rt)
    except Exception as e:  # noqa: BLE001 - any failure => agree on fallback collectively
        symm, err = None, f"{type(e).__name__}: {e}"
    # All ranks must agree, otherwise kernels would hang waiting on a missing peer.
    ok = [None] * rt.size
    dist.all_gather_object(ok, err, group=rt.cpu_group)
    bad = [(i, e) for i, e in enumerate(ok) if e is not None]
    if bad:
        if symm is not None:
            symm.close()
        rt.symm_failed = f"rank {bad[0][0]}: {bad[0][1]}"
        if rt.rank == 0:
            import warnings
            warnings.warn(
                "[b200dp] symmetric-memory runtime unavailable (" + rt.symm_failed +
                "); CUDA collectives FALL BACK to NCCL — this is not the product path.")
        return None
    rt.symm = symm
    if os.environ.get("HOROVOD_AUTOTUNE", "0") == "1":
        from .runtime import tuning
        try:
            res = tuning.autotune(symm)
            log.info("autotune: world %d -> %s", rt.size, res["table"])
        except Exception as e:  # noqa: BLE001 - keep the static table
            log.warning("autotune failed (%s); using the built-in algorithm table", e)
    return symm
