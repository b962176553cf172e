"""Python bindings (ctypes) for the in-tree sm_90a compute kernels
(``csrc/*.cu`` -> ``lib/libb200dp_kernels.so``).  Loaded lazily; every op registers itself
in ``_HAVE`` once its symbol resolves, so the functional layer can route per-op.
"""
from __future__ import annotations

import os
from typing import Dict

import torch

_HAVE: Dict[str, bool] = {}
_LIB = None
_TRIED = False


def _load():
    global _LIB, _TRIED
    if _TRIED:
        return _LIB
    _TRIED = True
    from ..runtime import lib as rtlib
    _LIB = rtlib.load_kernels()
    if _LIB is not None:
        from . import _bind
        _bind.register(_LIB, _HAVE)
    return _LIB


def enabled_for(x: torch.Tensor) -> bool:
    if not x.is_cuda or os.environ.get("B200DP_DISABLE_KERNELS", "0") == "1":
        return False
    if _load() is None:
        return False
    return torch.cuda.get_device_capability(x.device)[0] == 9


def has(op: str) -> bool:
    _load()
    return _HAVE.get(op, False)


def __getattr__(name):
    # op entry points live in _bind (populated when the library loads)
    from . import _bind
    if hasattr(_bind, name):
        return getattr(_bind, name)
    raise AttributeError(name)
