"""Fused NHWC BatchNorm(+residual)(+ReLU), max / average pooling (csrc/elementwise.cu) and the conv+BN+act unit
used by the ResNet blocks, whose convolution runs on the kernel ``ops.conv.kind`` chooses.

The batch-statistics reductions (here and in the producing GEMM / convolution epilogue) sum per-CTA
partials in a fixed order through one per-library set of slots, so they are bit-reproducible but must
not run concurrently on different CUDA streams; the training step issues them on one stream."""
from __future__ import annotations

import ctypes
import os
from typing import Optional

import torch
import torch.nn.functional as F

from . import counters
from . import grad_sink

_lib = None


def register(lib, have):
    global _lib
    if not hasattr(lib, "b200dp_bn_fwd"):
        return
    _lib = lib
    vp, i, f, ll, u64 = ctypes.c_void_p, ctypes.c_int, ctypes.c_float, ctypes.c_longlong, ctypes.c_uint64
    lib.b200dp_bn_fwd.argtypes = [vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, ll, i, f, f, i, i, i, vp, vp, u64]
    lib.b200dp_bn_apply.argtypes = [vp, vp, vp, vp, vp, ll, i, i, u64]
    lib.b200dp_bn_bwd.argtypes = [vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, i, ll, i, i, u64]
    lib.b200dp_bn_supported.argtypes = [i]
    if hasattr(lib, "b200dp_bn_fwd_sync"):
        lib.b200dp_bn_stats.argtypes = [vp, vp, ll, i, u64]
        lib.b200dp_bn_fwd_sync.argtypes = [vp] * 12 + [ll, vp, i, f, f, i, i, vp, u64]
        lib.b200dp_bn_bwd_reduce.argtypes = [vp, vp, vp, vp, vp, ll, i, i, u64]
        lib.b200dp_bn_bwd_apply.argtypes = [vp] * 10 + [ll, i, i, u64]
    lib.b200dp_ew_last_error.restype = ctypes.c_char_p
    have["bn_act"] = True
    have["conv_bn_act"] = True
    if hasattr(lib, "b200dp_stem_im2col"):
        lib.b200dp_stem_im2col.argtypes = [vp, vp, i, i, i, u64]
        have["stem_conv"] = True
    if hasattr(lib, "b200dp_avgpool_fwd"):
        lib.b200dp_avgpool_fwd.argtypes = [vp, vp, ctypes.c_longlong, i, i, u64]
        lib.b200dp_avgpool_bwd.argtypes = [vp, vp, ctypes.c_longlong, i, i, u64]
        have["global_avg_pool"] = True
    if hasattr(lib, "b200dp_maxpool_fwd"):
        lib.b200dp_maxpool_fwd.argtypes = [vp, vp, vp, i, i, i, i, u64]
        lib.b200dp_maxpool_bwd.argtypes = [vp, vp, vp, i, i, i, i, u64]
        have["max_pool_3x3_s2"] = True


def _ck(rc):
    if rc != 0:
        raise RuntimeError("elementwise kernel: " + (_lib.b200dp_ew_last_error() or b"").decode())


def _nhwc_ok(x: torch.Tensor) -> bool:
    """An activation the NHWC kernels take as it is: a dense channels_last bf16 CUDA tensor with a 16-byte
    aligned base."""
    return x.dim() == 4 and x.dtype == torch.bfloat16 and x.is_cuda and \
        x.is_contiguous(memory_format=torch.channels_last) and x.data_ptr() % 16 == 0


def bn_supported(x: torch.Tensor, C: int) -> bool:
    return _lib is not None and _nhwc_ok(x) and bool(_lib.b200dp_bn_supported(C))


def _cl(t: torch.Tensor) -> torch.Tensor:
    """``t`` as a dense channels_last tensor with a 16-byte aligned base (``contiguous`` keeps a dense view at an
    unaligned storage offset as it is)."""
    if t.is_contiguous(memory_format=torch.channels_last) and t.data_ptr() % 16 == 0:
        return t
    return t.clone(memory_format=torch.channels_last)


def params_ok(weight, bias, running_mean=None, running_var=None) -> bool:
    """The BN kernels read (and write back) gamma, beta and the running statistics in one dtype, chosen by gamma
    (``param_bf16``): gamma and beta must be present, and every one present must be a dense [C] tensor of that
    dtype, bf16 or fp32."""
    if weight is None or bias is None or weight.dtype not in (torch.bfloat16, torch.float32):
        return False
    C = weight.shape[0] if weight.dim() == 1 else -1
    return all(t.dtype == weight.dtype and t.device == weight.device and tuple(t.shape) == (C,) and t.stride(0) == 1
               for t in (weight, bias, running_mean, running_var) if t is not None)


def module_ok(bn, C: int, rows: int) -> bool:
    """Whether ``bn`` (a BatchNorm2d over ``C`` channels and ``rows`` = N H W positions) can run on the fused
    kernels: ``params_ok``; in training, a constant ``momentum`` (``None``, the cumulative average, takes torch's
    path) and more than one value per channel (torch refuses one); in eval mode, running statistics to apply."""
    if _lib is None or bn.num_features != C or not bool(_lib.b200dp_bn_supported(C)):
        return False
    if not params_ok(bn.weight, bn.bias, bn.running_mean, bn.running_var):
        return False
    if bn.training:
        return bn.momentum is not None and rows > 1
    return bn.track_running_stats and bn.running_mean is not None and bn.running_var is not None and rows > 0


def bn_forward(x, bn: torch.nn.BatchNorm2d, residual, relu: bool, stats_in=None, grads=(True, True)):
    """Training-mode BN(+residual)(+ReLU) of an NHWC bf16 ``x``; updates the running statistics and
    ``num_batches_tracked``.  ``stats_in``: the per-channel sums of ``x`` accumulated by the producing GEMM /
    conv epilogue (persistent buffer).  ``grads``: whether γ and β need gradients (their grad sinks count
    this use).  Returns ``(y, mask, ws)``: the ReLU sign bits (None without ReLU) and the per-channel
    ``(mean, invstd, a)`` that ``bn_backward`` reads."""
    N, C, H, W = x.shape
    M = N * H * W
    dev = x.device
    gamma, beta = bn.weight, bn.bias
    nbt = bn.num_batches_tracked if (bn.track_running_stats and bn.num_batches_tracked is not None
                                     and bn.num_batches_tracked.is_cuda) else None   # += 1 inside bn_finalize
    mom = bn.momentum                  # not None: module_ok sends the cumulative average to torch's path
    y = torch.empty_like(x, memory_format=torch.channels_last)
    ws = torch.empty(6 * C, dtype=torch.float32, device=dev)
    stats, mean, invstd, a, b = ws[:2 * C], ws[2 * C:3 * C], ws[3 * C:4 * C], ws[4 * C:5 * C], ws[5 * C:]
    if stats_in is not None:
        stats = stats_in
    pbf16 = int(gamma.dtype == torch.bfloat16)
    # ReLU sign bits, 1 byte per 8 channels: the backward reads 1/16th of what y would cost
    mask = torch.empty(M * (C // 8), dtype=torch.uint8, device=dev) if relu else None
    st = torch.cuda.current_stream(dev).cuda_stream
    _ck(_lib.b200dp_bn_fwd(x.data_ptr(), residual.data_ptr() if residual is not None else None,
                           y.data_ptr(), gamma.data_ptr(), beta.data_ptr(), stats.data_ptr(),
                           mean.data_ptr(), invstd.data_ptr(), a.data_ptr(), b.data_ptr(),
                           bn.running_mean.data_ptr() if bn.running_mean is not None else None,
                           bn.running_var.data_ptr() if bn.running_var is not None else None,
                           M, C, float(bn.eps), float(mom), int(relu), pbf16,
                           2 if stats_in is not None else 0,
                           mask.data_ptr() if mask is not None else None,
                           nbt.data_ptr() if nbt is not None else None, st))
    counters.bump("bn_fwd", 2 if stats_in is not None else 3)
    if grads[0]:
        grad_sink.note_forward(gamma)
    if grads[1]:
        grad_sink.note_forward(beta)
    return y, mask, (mean, invstd, a)


def bn_backward(dy, bn: torch.nn.BatchNorm2d, x, mask, ws, write_dres: bool = False):
    """Backward of ``bn_forward`` for a channels_last ``dy``.  ``mask``: ReLU sign bits applied to ``dy``
    (None: no ReLU).  ``write_dres``: also write the masked ``dy``, the gradient of the residual input.
    Returns ``(dx, dgamma, dbeta, dres)``; dgamma and dbeta are None when they went straight into the
    gradient buckets."""
    mean, invstd, a = ws
    N, C, H, W = x.shape
    M = N * H * W
    dx = torch.empty_like(x, memory_format=torch.channels_last)
    dres = torch.empty_like(x, memory_format=torch.channels_last) if write_dres else None
    sums = torch.empty(2 * C, dtype=torch.float32, device=x.device)
    # dgamma / dbeta: straight into the gradient-bucket slots when both parameters offer a sink
    gamma, beta = bn.weight, bn.bias
    gd, ga, gdone = grad_sink.begin(gamma)
    bd, ba, bdone = grad_sink.begin(beta)
    direct = gd is not None and bd is not None and not ga and not ba
    if direct:
        dg_ptr, db_ptr = gd.data_ptr(), bd.data_ptr()
    else:
        dgb = torch.empty(2 * C, dtype=gamma.dtype, device=x.device)
        dg_ptr, db_ptr = dgb.data_ptr(), dgb.data_ptr() + C * dgb.element_size()
    st = torch.cuda.current_stream(x.device).cuda_stream
    _ck(_lib.b200dp_bn_bwd(dy.data_ptr(), x.data_ptr(), mask.data_ptr() if mask is not None else None,
                           dx.data_ptr(), dres.data_ptr() if dres is not None else None,
                           a.data_ptr(), mean.data_ptr(), invstd.data_ptr(), sums.data_ptr(),
                           dg_ptr, db_ptr,
                           int(gamma.dtype == torch.bfloat16), M, C, int(mask is not None), st))
    counters.bump("bn_bwd", 2)
    if direct:
        gdone()
        bdone()
        return dx, None, None, dres
    return dx, dgb[:C], dgb[C:], dres                   # written by the kernel in the param dtype


class _BNActFn(torch.autograd.Function):
    """Training-mode BN over NHWC bf16 with fused residual add and ReLU."""

    @staticmethod
    def forward(ctx, x, gamma, beta, residual, relu, stats_in, bn):
        y, mask, ws = bn_forward(x, bn, residual, relu, stats_in, ctx.needs_input_grad[1:3])
        ctx.save_for_backward(x, mask, *ws)
        ctx.bn, ctx.has_res = bn, residual is not None
        return y

    @staticmethod
    def backward(ctx, dy):
        x, mask, *ws = ctx.saved_tensors
        dy = _cl(dy)
        dx, dgamma, dbeta, dres = bn_backward(dy, ctx.bn, x, mask, ws, write_dres=ctx.has_res and mask is not None)
        if ctx.has_res and dres is None:
            dres = dy                       # no ReLU: the residual branch gets dy unchanged
        return dx, dgamma, dbeta, dres, None, None, None


def bn_act(x, bn: torch.nn.BatchNorm2d, relu: bool, residual: Optional[torch.Tensor] = None,
           stats: Optional[torch.Tensor] = None):
    if residual is not None:
        residual = _cl(residual)
    if bn.training:
        return _BNActFn.apply(x, bn.weight, bn.bias, residual, relu, stats, bn)
    # inference: frozen statistics -> one fused apply pass
    a = (bn.weight.float() * torch.rsqrt(bn.running_var.float() + bn.eps))
    b = bn.bias.float() - bn.running_mean.float() * a
    y = torch.empty_like(x, memory_format=torch.channels_last)
    N, C, H, W = x.shape
    _ck(_lib.b200dp_bn_apply(x.data_ptr(), residual.data_ptr() if residual is not None else None,
                             y.data_ptr(), a.data_ptr(), b.data_ptr(), N * H * W, C, int(relu),
                             torch.cuda.current_stream(x.device).cuda_stream))
    counters.bump("bn_apply")
    return y


_FUSE_STATS = os.environ.get("B200DP_BN_STATS_IN_EPILOGUE", "1") == "1"


def _stats_buffer(bn, C: int, device):
    """Persistent per-BatchNorm accumulator (zero between steps: bn_finalize re-zeroes it after reading)."""
    buf = getattr(bn, "_b200dp_stats", None)
    if buf is None or buf.numel() != 2 * C or buf.device != device:
        buf = torch.zeros(2 * C, dtype=torch.float32, device=device)
        bn._b200dp_stats = buf
    return buf


def fused_stats(bn, C: int, device) -> Optional[torch.Tensor]:
    """The accumulator the producing conv / GEMM epilogue fills with the batch statistics of the BatchNorm
    that follows (no separate pass over its input), or None where that is not done."""
    return _stats_buffer(bn, C, device) if _FUSE_STATS and bn.training and C <= 2048 else None


def _out_shape(x, conv):
    """The shape [N, Cout, OH, OW] of the convolution's output."""
    N, _, H, W = x.shape
    (R, S), (sh, sw), (ph, pw), (dh, dw) = conv.kernel_size, conv.stride, conv.padding, conv.dilation
    return (N, conv.out_channels, max((H + 2 * ph - dh * (R - 1) - 1) // sh + 1, 0),
            max((W + 2 * pw - dw * (S - 1) - 1) // sw + 1, 0))


def _wants_grad(*ts) -> bool:
    return torch.is_grad_enabled() and any(t is not None and t.requires_grad for t in ts)


def conv_bn_act(x, conv, bn, relu: bool, residual=None):
    from . import conv as _conv
    C = conv.out_channels
    shape = _out_shape(x, conv) if x.dim() == 4 and isinstance(conv.padding, tuple) else None
    # eval mode: the fused apply pass is no autograd node, so only where nothing needs a gradient
    fused_bn = shape is not None and module_ok(bn, C, shape[0] * shape[2] * shape[3]) and \
        (residual is None or (residual.dtype == torch.bfloat16 and residual.shape == shape)) and \
        (bn.training or not _wants_grad(x, conv.weight, conv.bias, residual, bn.weight, bn.bias))
    # a kernel's output is a fresh NHWC bf16 tensor, which the fused BN takes: it consumes these statistics
    stats = fused_stats(bn, C, x.device) if fused_bn and _conv.kind(x, conv) is not None else None
    y = _conv.conv2d(x, conv, stats)
    if fused_bn and bn_supported(y, C):
        return bn_act(y, bn, relu, residual, stats=stats)
    y = bn(y)
    if residual is not None:
        y = y + residual
    return F.relu(y) if relu else y


class _MaxPoolFn(torch.autograd.Function):
    """3x3 / stride 2 / pad 1 max-pool on NHWC bf16 (byte arg-max saved; gather backward)."""

    @staticmethod
    def forward(ctx, x):
        N, C, H, W = x.shape
        OH, OW = (H - 1) // 2 + 1, (W - 1) // 2 + 1
        y = torch.empty((N, C, OH, OW), dtype=x.dtype, device=x.device,
                        memory_format=torch.channels_last)
        idx = torch.empty(N * OH * OW * C, dtype=torch.uint8, device=x.device)
        _ck(_lib.b200dp_maxpool_fwd(x.data_ptr(), y.data_ptr(), idx.data_ptr(), N, H, W, C,
                                    torch.cuda.current_stream(x.device).cuda_stream))
        counters.bump("maxpool_fwd")
        ctx.save_for_backward(idx)
        ctx.shape = (N, C, H, W)
        return y

    @staticmethod
    def backward(ctx, dy):
        (idx,) = ctx.saved_tensors
        N, C, H, W = ctx.shape
        if not dy.is_contiguous(memory_format=torch.channels_last):
            dy = dy.contiguous(memory_format=torch.channels_last)
        dx = torch.empty((N, C, H, W), dtype=dy.dtype, device=dy.device,
                         memory_format=torch.channels_last)
        _ck(_lib.b200dp_maxpool_bwd(dy.data_ptr(), idx.data_ptr(), dx.data_ptr(), N, H, W, C,
                                    torch.cuda.current_stream(dy.device).cuda_stream))
        counters.bump("maxpool_bwd")
        return dx


class _GlobalAvgPoolFn(torch.autograd.Function):
    """mean over H, W of an NHWC bf16 activation -> [N, C]; the backward is one broadcast write."""

    @staticmethod
    def forward(ctx, x):
        N, C, H, W = x.shape
        y = torch.empty((N, C), dtype=x.dtype, device=x.device)
        _ck(_lib.b200dp_avgpool_fwd(x.data_ptr(), y.data_ptr(), N, H * W, C,
                                    torch.cuda.current_stream(x.device).cuda_stream))
        counters.bump("avgpool_fwd")
        ctx.shape = (N, C, H, W)
        return y

    @staticmethod
    def backward(ctx, dy):
        N, C, H, W = ctx.shape
        dy = dy.contiguous()
        dx = torch.empty((N, C, H, W), dtype=dy.dtype, device=dy.device, memory_format=torch.channels_last)
        _ck(_lib.b200dp_avgpool_bwd(dy.data_ptr(), dx.data_ptr(), N, H * W, C,
                                    torch.cuda.current_stream(dy.device).cuda_stream))
        counters.bump("avgpool_bwd")
        return dx


def global_avg_pool(x):
    if _nhwc_ok(x) and x.shape[1] % 8 == 0 and hasattr(_lib, "b200dp_avgpool_fwd"):
        return _GlobalAvgPoolFn.apply(x)
    return x.mean(dim=(2, 3))


def max_pool_3x3_s2(x):
    if _nhwc_ok(x) and x.shape[1] % 8 == 0:
        return _MaxPoolFn.apply(x)
    return F.max_pool2d(x, kernel_size=3, stride=2, padding=1)
