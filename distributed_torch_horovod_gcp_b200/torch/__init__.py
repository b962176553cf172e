"""``import distributed_torch_horovod_gcp_b200.torch as hvd`` — the Horovod-shaped public API.

The reference uses exactly eight call sites of ``horovod.torch`` (app/torch_train.py:17,
210,217,227,232,249,259,266,308; SURVEY.md §2.3 A1–A8).  All of them, plus the rest of the
commonly used Horovod surface, are provided here on top of the H100 runtime.
"""
from __future__ import annotations

import os as _os

import torch as _torch

from .._state import (init, shutdown, is_initialized, rank, size, local_rank, local_size,
                      cross_rank, cross_size, is_homogeneous)
from .compression import Compression
from .mpi_ops import (Average, Sum, Adasum, Min, Max, Product, HorovodInternalError,
                      allreduce, allreduce_, allreduce_async, allreduce_async_,
                      grouped_allreduce, grouped_allreduce_, grouped_allreduce_async,
                      grouped_allreduce_async_,
                      allgather, allgather_async, grouped_allgather,
                      broadcast, broadcast_, broadcast_async, broadcast_async_,
                      alltoall, alltoall_async,
                      reducescatter, reducescatter_async, grouped_reducescatter,
                      synchronize, poll, barrier, join)
from .functions import (broadcast_parameters, broadcast_optimizer_state, broadcast_object,
                        allgather_object)
from .optimizer import DistributedOptimizer
from .optim import LARS, LAMB, Muon
from .sync_batch_norm import SyncBatchNorm
from .process_sets import ProcessSet, global_process_set, add_process_set, remove_process_set
from . import elastic


HostsUpdatedInterrupt = elastic.HostsUpdatedInterrupt   # raised by state.check_host_updates()


# ---------------------------------------------------------------- build / capability probes
def mpi_built() -> bool:
    return False


def mpi_enabled() -> bool:
    return False


def mpi_threads_supported() -> bool:
    return False


def gloo_built() -> bool:
    return True


def gloo_enabled() -> bool:
    return True


def nccl_built() -> int:
    """NCCL is present only as a fallback data plane; the product path is the sm_90a
    symmetric-memory kernels (see ``symm_built``)."""
    try:
        return int(_torch.distributed.is_nccl_available())
    except Exception:
        return 0


def cuda_built() -> bool:
    return _torch.version.cuda is not None


def rocm_built() -> bool:
    return False


def ddl_built() -> bool:
    return False


def ccl_built() -> bool:
    return False


def symm_built() -> bool:
    """True when the in-tree sm_90a runtime library has been built."""
    from ..runtime import lib
    return lib.available()


def symm_enabled() -> bool:
    """True when CUDA collectives are running on the symmetric-memory kernels."""
    from .. import _state
    return _state.runtime().symm is not None


# ---------------------------------------------------------------- timeline
def start_timeline(file_path: str, mark_cycles: bool = False) -> None:
    from .. import _state
    from ..utils.timeline import Timeline
    rt = _state._require_init()
    if rt.timeline is not None:
        rt.timeline.close()
    rt.timeline = Timeline(file_path, rt.rank)


def stop_timeline() -> None:
    from .. import _state
    rt = _state._require_init()
    if rt.timeline is not None:
        rt.timeline.close()
        rt.timeline = None


# ---------------------------------------------------------------- symmetric tensors
def symm_empty(numel: int, dtype=_torch.float32):
    """Allocate a flat tensor in NVSwitch-mapped symmetric memory (collective call).
    ``allreduce_`` / ``broadcast_`` on such a tensor run zero-copy."""
    from .. import _state
    symm = _state.get_symm()
    if symm is None:
        return _torch.empty(numel, dtype=dtype,
                            device="cuda" if _torch.cuda.is_available() else "cpu")
    return symm.alloc_tensor(numel, dtype)
