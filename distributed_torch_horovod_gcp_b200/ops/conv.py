"""Convolutions of NHWC bf16 activations on the sm_90a kernels.  ``kind`` is the one place that chooses a
convolution's kernel, and ``forward`` / ``dgrad`` / ``wgrad`` run each kind, for ``conv2d`` and for the ResNet
bottleneck node (ops/bottleneck.py):

- ``"gemm"``: a 1x1 stride-1 convolution is the wgmma GEMM (csrc/gemm_sm90.cu) on the NHWC rows (an NHWC
  activation is a row-major [N*H*W, C] matrix);
- ``"stem"``: the ResNet stem (7x7, stride 2, 3 input channels) is an im2col (csrc/elementwise.cu) + that GEMM;
- ``"implicit"``: 3x3 (stride 1/2, pad 1) and strided 1x1 convolutions run on the implicit-GEMM kernel
  (csrc/conv_sm90.cu), forward, data gradient and weight gradient, on the wgmma mainloop with the filter taps
  expressed as shifted 4D TMA boxes (zero padding = TMA out-of-bounds fill): no im2col buffer;
- anything else takes ``F.conv2d``.

Weights are consumed as ``[Cout][R][S][Cin]`` — PyTorch's ``channels_last`` layout of a
``[Cout, Cin, R, S]`` parameter — so ``model.to(memory_format=torch.channels_last)`` makes the
parameter itself the GEMM B operand; a parameter in the default layout is re-laid-out per call.

The weight-gradient kernels write the gradient in the weight's dtype themselves (split-K over pixels: the
last split to finish a tile sums the fp32 partials of all splits in split order, so the result is
bit-reproducible, and rounds once).  When the parameter carries a ``grad_sink`` (installed by the fused
engine) they write, or add, straight into the parameter's slot of the gradient bucket and the bucket
counter fires, so autograd's ``AccumulateGrad`` add/copy kernels disappear.  The stem's weight gradient is
summed in fp32 and returned to autograd.
"""
from __future__ import annotations

import ctypes
import os
from typing import Optional

import torch
import torch.nn.functional as F

from . import bn as _bn
from . import counters
from . import gemm as _gemm
from . import grad_sink

_lib = None
_USE_GEMM_1X1 = os.environ.get("B200DP_CONV1X1_GEMM", "1") == "1"
_USE_STEM_GEMM = os.environ.get("B200DP_STEM_GEMM", "1") == "1"
_ENABLED = os.environ.get("B200DP_CONV_KERNEL", "1") == "1"
STEM_KP = 168          # k = kh*24 + kw*3 + c (21 real + 3 zero-weighted columns per kernel row)


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


def kind(x: torch.Tensor, conv: torch.nn.Conv2d) -> Optional[str]:
    """Which kernel computes ``conv(x)``: ``"gemm"``, ``"stem"``, ``"implicit"`` (see the module docstring), or
    None for ``F.conv2d``.  Every kind takes a bf16 weight, no bias, one group and an NHWC bf16 ``x``
    (``ops.bn._nhwc_ok``).  ``B200DP_CONV1X1_GEMM=0`` / ``B200DP_STEM_GEMM=0`` / ``B200DP_CONV_KERNEL=0`` turn
    the first, second and third kind off; a 1x1 stride-1 convolution then takes the implicit-GEMM kernel."""
    w = conv.weight
    if conv.bias is not None or conv.groups != 1 or w.dtype != torch.bfloat16 or not _bn._nhwc_ok(x):
        return None
    Cout, Cin, R, S = w.shape
    H, W = x.shape[2], x.shape[3]
    if (_USE_GEMM_1X1 and _gemm._lib is not None and (R, S) == (1, 1) and conv.stride == (1, 1)
            and conv.padding == (0, 0) and Cout % 8 == 0 and Cin % 8 == 0):
        return "gemm"
    if (_USE_STEM_GEMM and _gemm._lib is not None and hasattr(_bn._lib, "b200dp_stem_im2col")
            and (R, S) == (7, 7) and conv.stride == (2, 2) and conv.padding == (3, 3) and Cin == 3
            and not x.requires_grad and H % 2 == 0 and W % 8 == 0 and Cout % 8 == 0):
        return "stem"
    p = (R - 1) // 2
    if (_ENABLED and _lib is not None and R == S and R in (1, 3) and conv.stride in ((1, 1), (2, 2))
            and conv.padding == (p, p) and conv.dilation == (1, 1) and Cin % 8 == 0 and Cout % 8 == 0
            and Cin >= 16 and (conv.stride == (1, 1) or (H % 2 == 0 and W % 2 == 0))):
        return "implicit"
    return None


def _rows(t: torch.Tensor) -> torch.Tensor:
    """A channels_last [N, C, H, W] activation as its [N*H*W, C] matrix (a view)."""
    N, C, H, W = t.shape
    return t.permute(0, 2, 3, 1).reshape(N * H * W, C)


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


def forward(x, weight, k: str, stride: int, pad: int, stats=None):
    """The forward launches of kind ``k``.  ``stats`` (fp32 [2*Cout], zero on entry): the epilogue adds the
    output's per-channel sum / sum of squares to it.  Returns the output (logical NCHW, NHWC memory), the
    weight as the kernel read it, and the activation the weight gradient reads: ``x``, or the stem's im2col
    matrix ([N*OH*OW, 168] bf16, about 1 GB at batch 256: kept rather than rebuilt, because HBM bandwidth, not
    an 80 GB H100's capacity, bounds the step)."""
    if k == "implicit":
        w = _krsc(weight)
        return conv_fprop(x, w, stride, pad, stats), w, x
    N, _, H, W = x.shape
    Cout = weight.shape[0]
    if k == "gemm":
        a, w = _rows(x), weight.reshape(Cout, x.shape[1])
    else:
        a = torch.empty((N * (H // 2) * (W // 2), STEM_KP), dtype=torch.bfloat16, device=x.device)
        _bn._ck(_bn._lib.b200dp_stem_im2col(x.data_ptr(), a.data_ptr(), N, H, W,
                                            torch.cuda.current_stream(x.device).cuda_stream))
        counters.bump("stem_im2col")
        w = torch.zeros((Cout, 7, 24), dtype=torch.bfloat16, device=x.device)
        w[:, :, :21] = weight.permute(0, 2, 3, 1).reshape(Cout, 7, 21)  # [Cout][kh][kw*3 + c]
        w = w.view(Cout, STEM_KP)
        H, W = H // 2, W // 2
    M, K = a.shape
    y = _gemm.gemm(a, w, torch.empty((M, Cout), dtype=torch.bfloat16, device=x.device), M, Cout, K, stats=stats)
    return y.view(N, H, W, Cout).permute(0, 3, 1, 2), w, (x if k == "gemm" else a)


def dgrad(dz, w, k: str, x_shape, stride: int, pad: int, residual=None, res_mask=None):
    """dx of kind ``k`` (not the stem, whose input needs no gradient) from the output gradient ``dz``, a dense
    channels_last tensor, and ``w`` as ``forward`` returned it.  GEMM only: ``residual`` (an activation of
    ``x_shape``) is added in the epilogue, kept only where the bits of ``res_mask`` are set."""
    if k == "implicit":
        return conv_dgrad(dz, w, x_shape, stride, pad)
    N, C, H, W = x_shape
    res = _rows(residual) if residual is not None else None
    return _gemm.dgrad(_rows(dz), w, res, res_mask).view(N, H, W, C).permute(0, 3, 1, 2)


def wgrad(dz, a, weight, k: str, stride: int, pad: int) -> Optional[torch.Tensor]:
    """dW of kind ``k`` in ``weight``'s shape from the output gradient ``dz`` and the activation ``a`` that
    ``forward`` returned, or ``None`` when it went straight into the weight's gradient-bucket slot."""
    if k == "implicit":
        return conv_wgrad(dz, a, weight, stride, pad)
    Cout = weight.shape[0]
    if k == "gemm":
        N, C, H, W = a.shape
        dw = _gemm.wgrad(_rows(dz), _rows(a), Cout, C, N * H * W, weight.dtype, owner=weight)
        return dw.view(weight.shape) if dw is not None else None
    M = a.shape[0]
    acc = torch.zeros((Cout, STEM_KP), dtype=torch.float32, device=dz.device)
    _gemm.gemm(_rows(dz), a, acc, Cout, STEM_KP, M, a_mn=True, b_mn=True, out_mode=1,
               splits=_gemm._splits_for(Cout, STEM_KP, M))
    dw = acc.view(Cout, 7, 24)[:, :, :21].reshape(Cout, 7, 7, 3).permute(0, 3, 1, 2).to(torch.bfloat16)
    return dw.contiguous(memory_format=torch.channels_last)


class _ConvFn(torch.autograd.Function):
    """A convolution on the kernels of kind ``k``."""

    @staticmethod
    def forward(ctx, x, weight, k, stride, pad, stats=None):
        if k != "stem" and ctx.needs_input_grad[1]:
            grad_sink.note_forward(weight)
        y, w, a = forward(x, weight, k, stride, pad, stats)
        ctx.save_for_backward(w, a)
        ctx.weight, ctx.k, ctx.stride, ctx.pad = weight, k, stride, pad
        return y

    @staticmethod
    def backward(ctx, dy):
        w, a = ctx.saved_tensors
        dy = _bn._cl(dy)
        dx = dw = None
        if ctx.needs_input_grad[0]:
            dx = dgrad(dy, w, ctx.k, a.shape, ctx.stride, ctx.pad)
        if ctx.needs_input_grad[1]:
            dw = wgrad(dy, a, ctx.weight, ctx.k, ctx.stride, ctx.pad)
        return dx, dw, None, None, None, None


def conv2d(x, conv: torch.nn.Conv2d, stats=None):
    """``conv(x)`` on the kernel ``kind`` chooses, else ``F.conv2d``.  ``stats`` (fp32 [2*Cout], zero on entry;
    taken only by a kernel kind): the epilogue adds the output's per-channel sum / sum of squares to it — the
    batch statistics of the BatchNorm that follows."""
    k = kind(x, conv)
    if k is None:
        b = conv.bias.to(x.dtype) if conv.bias is not None else None
        return F.conv2d(x, conv.weight.to(x.dtype), b, conv.stride, conv.padding, conv.dilation, conv.groups)
    return _ConvFn.apply(x, conv.weight, k, conv.stride[0], conv.padding[0], stats)


def conv2d_implicit(x: torch.Tensor, weight: torch.Tensor, stride: int = 1, padding: Optional[int] = None):
    """``F.conv2d`` of an NHWC bf16 activation and a raw weight on the implicit-GEMM kernel, for a shape ``kind``
    sends there."""
    if padding is None:
        padding = (weight.shape[2] - 1) // 2
    return _ConvFn.apply(x, weight, "implicit", int(stride), int(padding))


def conv3x3(x, weight, stride: int = 1):
    return conv2d_implicit(x, weight, stride, 1)
