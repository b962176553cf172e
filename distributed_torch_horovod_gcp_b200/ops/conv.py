"""Implicit-GEMM convolution binding (csrc/conv_sm90.cu): 3x3 (stride 1/2, pad 1) and 1x1
(stride 1/2) NHWC bf16 convolutions — forward, data gradient and weight gradient — on the
wgmma mainloop, with the filter taps expressed as shifted 4D TMA boxes (zero padding = TMA
out-of-bounds fill).  No cuDNN call and no im2col buffer on this path.

Weights are consumed as ``[Cout][R][S][Cin]`` — PyTorch's ``channels_last`` layout of a
``[Cout, Cin, R, S]`` parameter — so ``model.to(memory_format=torch.channels_last)`` makes the
parameter itself the GEMM B operand; a parameter in the default layout is re-laid-out per call.

The weight-gradient kernel writes the gradient in the weight's dtype itself (split-K over pixels: the
last split to finish a tile sums the fp32 partials of all splits in split order, so the result is
bit-reproducible, and rounds once).  When the parameter carries a ``grad_sink`` (installed by the fused
engine) it writes, or adds, straight into the parameter's slot of the gradient bucket and the bucket
counter fires, so autograd's ``AccumulateGrad`` add/copy kernels disappear.
"""
from __future__ import annotations

import ctypes
import os
from typing import Optional

import torch

from . import counters
from . import grad_sink

_lib = None
_ENABLED = os.environ.get("B200DP_CONV_KERNEL", "1") == "1"


def register(lib, have):
    global _lib
    if not hasattr(lib, "b200dp_conv_fprop"):
        return
    _lib = lib
    vp, i, u64 = ctypes.c_void_p, ctypes.c_int, ctypes.c_uint64
    lib.b200dp_conv_fprop.argtypes = [vp, vp, vp] + [i] * 11 + [vp, u64]
    lib.b200dp_conv_dgrad.argtypes = [vp, vp, vp] + [i] * 11 + [u64]
    lib.b200dp_conv_wgrad.argtypes = [vp, vp, vp] + [i] * 14 + [u64]
    lib.b200dp_conv_last_error.restype = ctypes.c_char_p
    have["conv3x3"] = True
    have["conv_implicit_gemm"] = True


def _ck(rc):
    if rc != 0:
        raise RuntimeError("conv kernel: " + (_lib.b200dp_conv_last_error() or b"").decode())


def _nhwc(x: torch.Tensor) -> bool:
    return x.dim() == 4 and x.dtype == torch.bfloat16 and x.is_cuda and \
        x.is_contiguous(memory_format=torch.channels_last) and x.data_ptr() % 16 == 0


def supported(x: torch.Tensor, weight: torch.Tensor, stride, padding, dilation=(1, 1), groups=1) -> bool:
    if _lib is None or not _ENABLED or weight.dtype != torch.bfloat16 or not _nhwc(x):
        return False
    Cout, Cin, R, S = weight.shape
    sh, sw = (stride, stride) if isinstance(stride, int) else tuple(stride)
    ph, pw = (padding, padding) if isinstance(padding, int) else tuple(padding)
    dil = (dilation, dilation) if isinstance(dilation, int) else tuple(dilation)
    if groups != 1 or dil != (1, 1) or sh != sw or ph != pw or R != S or R not in (1, 3):
        return False
    if ph != (R - 1) // 2 or sh not in (1, 2) or Cin % 8 or Cout % 8 or Cin < 16:
        return False
    if sh == 2 and (x.shape[2] % 2 or x.shape[3] % 2):
        return False
    return True


def _krsc(weight: torch.Tensor) -> torch.Tensor:
    if weight.is_contiguous(memory_format=torch.channels_last) and weight.data_ptr() % 16 == 0:
        return weight
    return weight.contiguous(memory_format=torch.channels_last)


def conv_fprop(x, w_krsc, stride: int, pad: int, stats=None):
    N, Cin, H, W = x.shape
    Cout, _, R, S = w_krsc.shape
    y = torch.empty((N, Cout, H // stride, W // stride), dtype=torch.bfloat16, device=x.device,
                    memory_format=torch.channels_last)
    _ck(_lib.b200dp_conv_fprop(x.data_ptr(), w_krsc.data_ptr(), y.data_ptr(), N, H, W, Cin, Cout, R, S,
                               stride, pad, 0, 0, stats.data_ptr() if stats is not None else None,
                               torch.cuda.current_stream(x.device).cuda_stream))
    counters.bump("conv_fprop")
    return y


def conv_dgrad(dy, w_krsc, x_shape, stride: int, pad: int):
    N, Cin, H, W = x_shape
    Cout, _, R, S = w_krsc.shape
    dx = torch.empty((N, Cin, H, W), dtype=torch.bfloat16, device=dy.device,
                     memory_format=torch.channels_last)
    _ck(_lib.b200dp_conv_dgrad(dy.data_ptr(), w_krsc.data_ptr(), dx.data_ptr(), N, H, W, Cin, Cout, R, S,
                               stride, pad, 0, 0, torch.cuda.current_stream(dy.device).cuda_stream))
    counters.bump("conv_dgrad", 2 if (R == 1 and stride == 2) else 1)
    return dx


def conv_wgrad(dy, x, weight, stride: int, pad: int) -> Optional[torch.Tensor]:
    """Returns dW in the weight's layout, or ``None`` when it was written into the gradient bucket."""
    N, Cin, H, W = x.shape
    Cout, _, R, S = weight.shape
    # the kernel writes [Cout][R][S][Cin]: the channels_last order of the weight
    dst, acc, done = grad_sink.begin(weight, krsc=True)
    ret = None
    if dst is None:
        dst = torch.empty_like(weight, memory_format=torch.channels_last)
        acc, ret = False, dst
    _ck(_lib.b200dp_conv_wgrad(dy.data_ptr(), x.data_ptr(), dst.data_ptr(), N, H, W, Cin, Cout, R, S,
                               stride, pad, 0, 0, 0, int(acc), int(dst.dtype == torch.bfloat16),
                               torch.cuda.current_stream(dy.device).cuda_stream))
    counters.bump("conv_wgrad", 1)
    if done is not None:
        done()
    return ret


class _ConvFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, weight, stride, pad, stats=None):
        w = _krsc(weight)
        if ctx.needs_input_grad[1]:
            grad_sink.note_forward(weight)
        y = conv_fprop(x, w, stride, pad, stats)
        ctx.save_for_backward(x, w)
        ctx.weight = weight
        ctx.stride, ctx.pad = stride, pad
        return y

    @staticmethod
    def backward(ctx, dy):
        x, w = ctx.saved_tensors
        if not dy.is_contiguous(memory_format=torch.channels_last) or dy.data_ptr() % 16:
            dy = dy.contiguous(memory_format=torch.channels_last)
        dx = dw = None
        if ctx.needs_input_grad[0]:
            dx = conv_dgrad(dy, w, x.shape, ctx.stride, ctx.pad)
        if ctx.needs_input_grad[1]:
            dw = conv_wgrad(dy, x, ctx.weight, ctx.stride, ctx.pad)
        return dx, dw, None, None, None


def conv2d(x: torch.Tensor, weight: torch.Tensor, stride: int = 1, padding: Optional[int] = None, stats=None):
    """``F.conv2d`` for NHWC bf16 activations on the sm_90a implicit-GEMM kernel.  ``stats`` (fp32
    [2*Cout], zero on entry): the kernel's epilogue adds the per-channel sum / sum of squares of the
    output to it — the batch statistics of the BatchNorm that follows."""
    if padding is None:
        padding = (weight.shape[2] - 1) // 2
    return _ConvFn.apply(x, weight, int(stride), int(padding), stats)


def conv3x3(x, weight, stride: int = 1):
    return conv2d(x, weight, stride, 1)
