"""Fused dropout + residual add binding (``dropout_add_kernel`` in csrc/elementwise.cu), bf16:
``out = residual + keep * y / q`` with one keep bit per element of ``y`` (``residual=None``: plain dropout).

The keep bits come from Philox4x32-10 (the mapping is in the kernel's comment) under a seed that torch's CUDA
generator draws into device memory on every call, as for the attention dropout (ops/attention.py):
``torch.manual_seed`` reproduces the masks and each replay of a captured CUDA graph draws new ones.  The
keep probability is ``q = round((1 - p) 2^16) / 2^16`` and kept elements are scaled by exactly ``1 / q``.  The
backward regenerates the bits from the saved seed (nothing per element is saved):
``dy = keep * dout / q`` by the same kernel, and ``dresidual = dout``."""
from __future__ import annotations

import ctypes

import torch

from . import counters

_lib = None


def register(lib, have):
    global _lib
    if not hasattr(lib, "b200dp_dropout_add"):
        return
    _lib = lib
    vp = ctypes.c_void_p
    lib.b200dp_dropout_add.argtypes = [vp, vp, vp, ctypes.c_longlong, vp, ctypes.c_float, ctypes.c_uint64]
    lib.b200dp_ew_last_error.restype = ctypes.c_char_p
    have["dropout_add"] = True


def _ok(t: torch.Tensor) -> bool:
    return t.dtype == torch.bfloat16 and t.is_contiguous() and t.numel() % 8 == 0 and t.data_ptr() % 16 == 0


def supported(y, residual) -> bool:
    return _lib is not None and y.is_cuda and _ok(y) and (
        residual is None or (residual.device == y.device and residual.shape == y.shape and _ok(residual)))


def _launch(y, residual, out, seed, p):
    rc = _lib.b200dp_dropout_add(y.data_ptr(), None if residual is None else residual.data_ptr(), out.data_ptr(),
                                 y.numel(), seed.data_ptr(), p, torch.cuda.current_stream(y.device).cuda_stream)
    if rc != 0:
        raise RuntimeError("dropout_add kernel: " + (_lib.b200dp_ew_last_error() or b"").decode())
    counters.bump("dropout_add")


class _DropoutAddFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, y, residual, p):
        seed = torch.randint(0, 2 ** 62, (2,), dtype=torch.int64, device=y.device)   # Philox key, offset
        out = torch.empty_like(y)
        _launch(y, residual, out, seed, p)
        ctx.save_for_backward(seed)
        ctx.p = p
        ctx.has_residual = residual is not None
        return out

    @staticmethod
    def backward(ctx, dout):
        (seed,) = ctx.saved_tensors
        dout = dout.contiguous()
        dy = torch.empty_like(dout)
        _launch(dout, None, dy, seed, ctx.p)
        return dy, (dout if ctx.has_residual else None), None


def dropout_add(y, residual, p: float):
    """``residual + dropout(y, p)`` (``residual=None``: ``dropout(y, p)``) for 0 < p <= 1 on supported inputs."""
    return _DropoutAddFn.apply(y, residual, float(p))
