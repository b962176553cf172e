"""Locate / load the in-tree native libraries.

  lib/libb200dp_comm.so     C++ runtime (csrc/runtime.cpp: symmetric heap, fd passing) +
                            sm_90a comm kernels (csrc/comm_kernels.cu: allreduce/broadcast(+optimizer))
  lib/libb200dp_kernels.so  sm_90a math  (csrc/gemm_sm90.cu …)  — wgmma GEMM, BN, LSTM …

They are built IN-TREE by ``build.py`` (``__graft_entry__.build()``) so they travel with the
repo snapshot to the GPU box, and loaded with ctypes (no torch headers => seconds to build).
On a CUDA machine a missing library is an ERROR unless ``B200DP_ALLOW_FALLBACK=1``: tests
must not silently pass on a PyTorch fallback.
"""
from __future__ import annotations

import ctypes
import os
from typing import Optional

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_DIR = os.path.join(os.path.dirname(_HERE), "lib")
_cache = {}


def _path(name: str) -> str:
    return os.path.join(LIB_DIR, name)


def available(name: str = "libb200dp_comm.so") -> bool:
    return os.path.exists(_path(name))


def _load(name: str) -> Optional[ctypes.CDLL]:
    if name in _cache:
        return _cache[name]
    p = _path(name)
    lib = None
    if not os.path.exists(p) and os.environ.get("B200DP_NO_AUTOBUILD", "0") != "1":
        # fresh checkout (the .so files are git-ignored): build in-tree once, if nvcc is present
        try:
            import torch
            if torch.cuda.is_available():
                from .. import build as _build
                _build.build()
        except Exception as e:  # noqa: BLE001 - reported below if the library is still missing
            import warnings
            warnings.warn(f"[b200dp] in-tree native build failed: {e}")
    if os.path.exists(p):
        lib = ctypes.CDLL(p, mode=ctypes.RTLD_GLOBAL)
    else:
        import torch
        if torch.cuda.is_available() and os.environ.get("B200DP_ALLOW_FALLBACK", "0") != "1":
            raise RuntimeError(
                f"native library {p} is missing on a CUDA machine; run "
                f"`python -c 'import __graft_entry__ as g; g.build()'` (or set "
                f"B200DP_ALLOW_FALLBACK=1 to accept the PyTorch/NCCL fallback)")
    _cache[name] = lib
    return lib


def load_comm() -> Optional[ctypes.CDLL]:
    return _load("libb200dp_comm.so")


def load_kernels() -> Optional[ctypes.CDLL]:
    return _load("libb200dp_kernels.so")
