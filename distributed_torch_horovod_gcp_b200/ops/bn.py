"""Fused NHWC BatchNorm(+residual)(+ReLU) (csrc/elementwise.cu) and the conv+BN+act unit used by
the ResNet blocks.  1x1 stride-1 convolutions run on the wgmma GEMM (an NHWC activation is a
row-major [N*H*W, C] matrix), the 7x7 stem on im2col + that GEMM, and 3x3 / strided 1x1 convolutions
on the implicit-GEMM kernel (ops/conv.py, csrc/conv_sm90.cu); cuDNN is only the fallback for shapes
none of these cover (e.g. a 3-channel 3x3 stem).

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
from . import gemm as _gemm
from . import grad_sink

_lib = None
_USE_GEMM_1X1 = os.environ.get("B200DP_CONV1X1_GEMM", "1") == "1"


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
        d = ctypes.c_double
        lib.b200dp_bn_stats.argtypes = [vp, vp, ll, i, u64]
        lib.b200dp_bn_fwd_sync.argtypes = [vp] * 12 + [ll, d, i, f, f, i, i, vp, u64]
        lib.b200dp_bn_bwd_reduce.argtypes = [vp, vp, vp, vp, vp, ll, i, i, u64]
        lib.b200dp_bn_bwd_apply.argtypes = [vp] * 9 + [d, ll, i, i, u64]
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
    return x.dim() == 4 and x.dtype == torch.bfloat16 and \
        x.is_contiguous(memory_format=torch.channels_last) and x.data_ptr() % 16 == 0


def bn_supported(x: torch.Tensor, C: int) -> bool:
    return _lib is not None and _nhwc_ok(x) and bool(_lib.b200dp_bn_supported(C))


class _BNActFn(torch.autograd.Function):
    """Training-mode BN over NHWC bf16 with fused residual add and ReLU."""

    @staticmethod
    def forward(ctx, x, gamma, beta, running_mean, running_var, residual, relu, eps, momentum,
                stats_in=None, box=None, nbt=None):
        N, C, H, W = x.shape
        M = N * H * W
        dev = x.device
        y = torch.empty_like(x, memory_format=torch.channels_last)
        ws = torch.empty(6 * C, dtype=torch.float32, device=dev)
        stats, mean, invstd, a, b = ws[:2 * C], ws[2 * C:3 * C], ws[3 * C:4 * C], ws[4 * C:5 * C], ws[5 * C:]
        if stats_in is not None:
            stats = stats_in              # accumulated by the producing GEMM / conv epilogue (persistent buffer)
        pbf16 = int(gamma.dtype == torch.bfloat16)
        # ReLU sign bits, 1 byte per 8 channels: the backward reads 1/16th of what y would cost
        mask = torch.empty(M * (C // 8), dtype=torch.uint8, device=dev) if relu else None
        st = torch.cuda.current_stream(dev).cuda_stream
        _ck(_lib.b200dp_bn_fwd(x.data_ptr(), residual.data_ptr() if residual is not None else None,
                               y.data_ptr(), gamma.data_ptr(), beta.data_ptr(), stats.data_ptr(),
                               mean.data_ptr(), invstd.data_ptr(), a.data_ptr(), b.data_ptr(),
                               running_mean.data_ptr() if running_mean is not None else None,
                               running_var.data_ptr() if running_var is not None else None,
                               M, C, float(eps), float(momentum), int(relu), pbf16,
                               2 if stats_in is not None else 0,
                               mask.data_ptr() if mask is not None else None,
                               nbt.data_ptr() if nbt is not None else None, st))
        counters.bump("bn_fwd", 2 if stats_in is not None else 3)
        ctx.save_for_backward(x, mask, mean, invstd, a)
        ctx.relu, ctx.has_res, ctx.pdtype = relu, residual is not None, gamma.dtype
        ctx.affine = (gamma, beta)
        ctx.box = box
        if box is not None and residual is None and not relu and ctx.needs_input_grad[0]:
            box.armed = box.want_mask = True      # consumer role (see backward)
        if ctx.needs_input_grad[1]:
            grad_sink.note_forward(gamma)
        if ctx.needs_input_grad[2]:
            grad_sink.note_forward(beta)
        return y

    @staticmethod
    def backward(ctx, dy):
        x, mask, mean, invstd, a = ctx.saved_tensors
        N, C, H, W = x.shape
        M = N * H * W
        if not dy.is_contiguous(memory_format=torch.channels_last):
            dy = dy.contiguous(memory_format=torch.channels_last)
        dx = torch.empty_like(x, memory_format=torch.channels_last)
        box = ctx.box
        relu = ctx.relu
        if box is not None and not ctx.has_res and not relu and box.ext_mask is not None:
            # downsample BN of a projection block: ``dy`` is the block-output gradient BEFORE the block's
            # final ReLU mask, whose sign bits the block's BN+add+ReLU backward left in the box
            ext_mask, box.ext_mask = box.ext_mask, None
            assert ext_mask.numel() == M * (C // 8)
            mask, relu = ext_mask, True
        # the masked skip gradient is only materialised when nobody downstream applies the sign bits itself
        hand_off = ctx.has_res and ctx.relu and box is not None and box.armed and not box.consumed
        dres = torch.empty_like(x, memory_format=torch.channels_last) if (ctx.has_res and ctx.relu and not hand_off) \
            else None
        sums = torch.empty(2 * C, dtype=torch.float32, device=x.device)
        # dgamma / dbeta: straight into the gradient-bucket slots when both parameters offer a sink
        gamma, beta = ctx.affine
        gd, ga, gdone = grad_sink.begin(gamma)
        bd, ba, bdone = grad_sink.begin(beta)
        direct = gd is not None and bd is not None and not ga and not ba
        if direct:
            dg_ptr, db_ptr = gd.data_ptr(), bd.data_ptr()
        else:
            dgb = torch.empty(2 * C, dtype=ctx.pdtype, device=x.device)
            dg_ptr, db_ptr = dgb.data_ptr(), dgb.data_ptr() + C * dgb.element_size()
        st = torch.cuda.current_stream(x.device).cuda_stream
        _ck(_lib.b200dp_bn_bwd(dy.data_ptr(), x.data_ptr(), mask.data_ptr() if mask is not None else None,
                               dx.data_ptr(), dres.data_ptr() if dres is not None else None,
                               a.data_ptr(), mean.data_ptr(), invstd.data_ptr(), sums.data_ptr(),
                               dg_ptr, db_ptr,
                               int(ctx.pdtype == torch.bfloat16), M, C, int(relu), st))
        counters.bump("bn_bwd", 2)
        if direct:
            dgamma = dbeta = None
            gdone()
            bdone()
        else:
            dgamma, dbeta = dgb[:C], dgb[C:]              # written by the kernel in the param dtype
        if hand_off:
            if box.want_mask:
                box.ext_mask = mask         # projection block: the downsample BN backward masks dy itself
                dres = dy
            else:
                box.park(dy, mask)          # identity block: conv1's dgrad epilogue adds mask(dy)
                dres = None
        elif ctx.has_res and dres is None:
            dres = dy                       # no ReLU: the residual branch gets dy unchanged
            if box is not None and not box.want_mask and box.park(dres):
                dres = None
        return dx, dgamma, dbeta, None, None, dres, None, None, None, None, None, None


def bn_act(x, bn: torch.nn.BatchNorm2d, relu: bool, residual: Optional[torch.Tensor] = None,
           stats: Optional[torch.Tensor] = None, box=None):
    if residual is not None and not residual.is_contiguous(memory_format=torch.channels_last):
        residual = residual.contiguous(memory_format=torch.channels_last)
    if bn.training:
        nbt = bn.num_batches_tracked if (bn.track_running_stats and bn.num_batches_tracked is not None
                                         and bn.num_batches_tracked.is_cuda) else None   # += 1 inside bn_finalize
        mom = bn.momentum if bn.momentum is not None else 0.1
        return _BNActFn.apply(x, bn.weight, bn.bias, bn.running_mean, bn.running_var, residual,
                              relu, bn.eps, mom, stats, box, nbt)
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


def _is_gemm_conv(x, conv) -> bool:
    w = conv.weight
    return (_USE_GEMM_1X1 and _gemm._lib is not None and conv.kernel_size == (1, 1)
            and conv.stride == (1, 1) and conv.padding == (0, 0) and conv.groups == 1
            and conv.bias is None and w.dtype == torch.bfloat16 and _nhwc_ok(x)
            and w.shape[0] % 8 == 0 and w.shape[1] % 8 == 0)


_USE_STEM_GEMM = os.environ.get("B200DP_STEM_GEMM", "1") == "1"
STEM_KP = 168          # k = kh*24 + kw*3 + c (21 real + 3 zero-weighted columns per kernel row)


class _StemConvFn(torch.autograd.Function):
    """ResNet stem (7x7, stride 2, pad 3, 3 input channels) as im2col + wgmma GEMM.  The im2col
    matrix ([N*112*112, 168] bf16, about 1 GB at batch 256) is kept for the weight gradient instead
    of being rebuilt: it fits easily in an 80 GB H100, and HBM bandwidth, not capacity, bounds
    the step."""

    @staticmethod
    def forward(ctx, x, weight, stats=None):
        N, C, H, W = x.shape
        OH, OW = H // 2, W // 2
        M = N * OH * OW
        cols = torch.empty((M, STEM_KP), dtype=torch.bfloat16, device=x.device)
        _ck(_lib.b200dp_stem_im2col(x.data_ptr(), cols.data_ptr(), N, H, W,
                                    torch.cuda.current_stream(x.device).cuda_stream))
        counters.bump("stem_im2col")
        Cout = weight.shape[0]
        wp = torch.zeros((Cout, 7, 24), dtype=torch.bfloat16, device=x.device)
        wp[:, :, :21] = weight.permute(0, 2, 3, 1).reshape(Cout, 7, 21)  # [Cout][kh][kw*3 + c]
        wp = wp.view(Cout, STEM_KP)
        y = torch.empty((M, Cout), dtype=torch.bfloat16, device=x.device)
        _gemm.gemm(cols, wp, y, M, Cout, STEM_KP, stats=stats)
        ctx.save_for_backward(cols)
        ctx.wshape = weight.shape
        return y.view(N, OH, OW, Cout).permute(0, 3, 1, 2)

    @staticmethod
    def backward(ctx, dy):
        (cols,) = ctx.saved_tensors
        Cout = ctx.wshape[0]
        M = cols.shape[0]
        dy2 = dy.permute(0, 2, 3, 1).reshape(M, Cout)
        if not dy2.is_contiguous():
            dy2 = dy2.contiguous()
        acc = torch.zeros((Cout, STEM_KP), dtype=torch.float32, device=dy.device)
        _gemm.gemm(dy2, cols, acc, Cout, STEM_KP, M, a_mn=True, b_mn=True, out_mode=1,
                   splits=_gemm._splits_for(Cout, STEM_KP, M))
        dw = acc.view(Cout, 7, 24)[:, :, :21].reshape(Cout, 7, 7, 3).permute(0, 3, 1, 2).to(torch.bfloat16)
        return None, dw.contiguous(memory_format=torch.channels_last), None


def _is_stem_conv(x, conv) -> bool:
    return (_USE_STEM_GEMM and _gemm._lib is not None and hasattr(_lib, "b200dp_stem_im2col")
            and conv.kernel_size == (7, 7) and conv.stride == (2, 2) and conv.padding == (3, 3)
            and conv.groups == 1 and conv.bias is None and conv.in_channels == 3
            and conv.weight.dtype == torch.bfloat16 and _nhwc_ok(x) and not x.requires_grad
            and x.shape[2] % 2 == 0 and x.shape[3] % 8 == 0 and conv.out_channels % 8 == 0)


_FUSE_STATS = os.environ.get("B200DP_BN_STATS_IN_EPILOGUE", "1") == "1"


def conv2d(x, conv: torch.nn.Conv2d, box=None, stats=None, park=None):
    """Convolution of an NHWC bf16 activation; 1x1/stride-1 and the 7x7 stem -> wgmma GEMM, 3x3 and
    strided 1x1 -> implicit-GEMM kernel.  Returns ``(y, stats_filled)``: when ``stats`` (fp32 [2*Cout]
    accumulator) is given and the kernel that ran supports it, its epilogue has added the output's
    per-channel sum / sum of squares."""
    w = conv.weight
    if _is_gemm_conv(x, conv):
        N, C, H, W = x.shape
        x2 = x.permute(0, 2, 3, 1).reshape(N * H * W, C)             # view: NHWC rows
        y2 = _gemm.linear(x2, w.reshape(w.shape[0], C), owner=w, box=box, stats=stats, park=park)     # [M, Cout]
        return y2.view(N, H, W, w.shape[0]).permute(0, 3, 1, 2), stats is not None   # logical NCHW, NHWC memory
    if _is_stem_conv(x, conv):
        return _StemConvFn.apply(x, w, stats), stats is not None
    from . import conv as _conv
    if conv.bias is None and _conv.supported(x, w, conv.stride, conv.padding, conv.dilation, conv.groups):
        return _conv.conv2d(x, w, conv.stride[0], conv.padding[0], stats, park), stats is not None
    return F.conv2d(x, w, conv.bias, conv.stride, conv.padding, conv.dilation, conv.groups), False


def _stats_buffer(bn, C: int, device):
    """Persistent per-BatchNorm accumulator (zero between steps: bn_finalize re-zeroes it after reading)."""
    buf = getattr(bn, "_b200dp_stats", None)
    if buf is None or buf.numel() != 2 * C or buf.device != device:
        buf = torch.zeros(2 * C, dtype=torch.float32, device=device)
        bn._b200dp_stats = buf
    return buf


def conv_bn_act(x, conv, bn, relu: bool, residual=None, skip_box=None, input_box=None, park_box=None):
    """``input_box``: this conv consumes the block input whose skip gradient will arrive through the
    box; ``skip_box``: this BN's residual IS that block input, or (projection block) this BN is the
    downsample BN / the block's last BN exchanging the ReLU sign bits; ``park_box``: this conv's input
    gradient is handed to the box's consumer instead of being returned (grad_sink.GradBox)."""
    C = conv.out_channels
    fused_bn = _lib is not None and bn.weight is not None and bool(_lib.b200dp_bn_supported(C)) and \
        (residual is None or residual.dtype == torch.bfloat16)
    # batch statistics come out of the conv / GEMM epilogue (no separate pass over y)
    want_stats = _FUSE_STATS and fused_bn and bn.training and C <= 2048 and x.dtype == torch.bfloat16
    stats = _stats_buffer(bn, C, x.device) if want_stats else None
    y, filled = conv2d(x, conv, box=input_box, stats=stats, park=park_box)
    if stats is not None and not filled:
        stats = None
    if fused_bn and bn_supported(y, C):
        return bn_act(y, bn, relu, residual, stats=stats, box=skip_box)
    if stats is not None:
        stats.zero_()          # filled but not consumed by the fused BN: keep the accumulator clean
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
