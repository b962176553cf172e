"""Fused LayerNorm forward/backward (csrc/elementwise.cu: ln_fwd / ln_bwd), bf16 in/out, fp32
statistics; the backward computes dx and the gamma/beta column reductions in one pass."""
from __future__ import annotations

import ctypes

import torch

from . import counters

_lib = None


def register(lib, have):
    global _lib
    if not hasattr(lib, "b200dp_ln_fwd"):
        return
    _lib = lib
    vp, i, f, ll, u64 = ctypes.c_void_p, ctypes.c_int, ctypes.c_float, ctypes.c_longlong, ctypes.c_uint64
    lib.b200dp_ln_fwd.argtypes = [vp, vp, vp, vp, vp, vp, ll, i, f, i, u64]
    lib.b200dp_ln_bwd.argtypes = [vp, vp, vp, vp, vp, vp, vp, vp, vp, ll, i, i, u64]
    lib.b200dp_ln_supported.argtypes = [i]
    have["layer_norm"] = True


def supported(x: torch.Tensor, weight, bias) -> bool:
    """bf16 ``x`` with at least one row and a 16-byte aligned base (the kernels load it in 16-byte vectors), and
    gamma and beta of C elements in one dtype, bf16 or fp32 (the kernels read both in the dtype ``pbf16`` names)."""
    if _lib is None or weight is None or bias is None or x.dim() < 1:
        return False
    C = x.shape[-1]
    return (x.dtype == torch.bfloat16 and x.is_cuda and x.numel() > 0 and x.data_ptr() % 16 == 0
            and weight.dtype in (torch.bfloat16, torch.float32) and bias.dtype == weight.dtype
            and tuple(weight.shape) == (C,) and tuple(bias.shape) == (C,) and weight.stride(0) == 1
            and bias.stride(0) == 1 and weight.device == x.device and bias.device == x.device
            and bool(_lib.b200dp_ln_supported(C)))


class _LayerNormFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, weight, bias, eps):
        C = x.shape[-1]
        x2 = x.reshape(-1, C)
        if not x2.is_contiguous():
            x2 = x2.contiguous()
        R = x2.shape[0]
        y = torch.empty_like(x2)
        stats = torch.empty(2 * R, dtype=torch.float32, device=x.device)
        pbf16 = int(weight.dtype == torch.bfloat16)
        rc = _lib.b200dp_ln_fwd(x2.data_ptr(), y.data_ptr(), weight.data_ptr(), bias.data_ptr(),
                                stats.data_ptr(), stats.data_ptr() + 4 * R, R, C, float(eps), pbf16,
                                torch.cuda.current_stream(x.device).cuda_stream)
        if rc != 0:
            raise RuntimeError("ln_fwd failed")
        counters.bump("ln_fwd")
        ctx.save_for_backward(x2, weight, stats)
        ctx.shape, ctx.pbf16 = x.shape, pbf16
        return y.view(x.shape)

    @staticmethod
    def backward(ctx, dy):
        x2, weight, stats = ctx.saved_tensors
        R, C = x2.shape
        dy2 = dy.reshape(R, C)
        if not dy2.is_contiguous() or dy2.data_ptr() % 16:
            dy2 = dy2.clone(memory_format=torch.contiguous_format)
        dx = torch.empty_like(x2)
        sums = torch.empty(2 * C, dtype=torch.float32, device=dy.device)
        dgb = torch.empty(2 * C, dtype=weight.dtype, device=dy.device)
        rc = _lib.b200dp_ln_bwd(dy2.data_ptr(), x2.data_ptr(), dx.data_ptr(), weight.data_ptr(),
                                stats.data_ptr(), stats.data_ptr() + 4 * R, sums.data_ptr(),
                                dgb.data_ptr(), dgb.data_ptr() + C * dgb.element_size(), R, C,
                                ctx.pbf16, torch.cuda.current_stream(dy.device).cuda_stream)
        if rc != 0:
            raise RuntimeError("ln_bwd failed")
        counters.bump("ln_bwd", 2)
        return dx.view(ctx.shape), dgb[:C], dgb[C:], None


def layer_norm(x, weight, bias, eps: float = 1e-6):
    return _LayerNormFn.apply(x, weight, bias, eps)
