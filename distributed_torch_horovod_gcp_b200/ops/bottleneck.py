"""ResNet bottleneck block (``models.resnet.Bottleneck``) as ONE autograd node on the kernel path.

The block input feeds conv1 and the skip connection, so its gradient is the sum of two activation-sized
tensors.  The backward adds the skip gradient in conv1's dgrad GEMM epilogue (``dx = dz @ W + residual``)
instead of a stand-alone ``add`` kernel, and bn3 writes no masked copy of its incoming gradient ``dy``:
identity block: the residual is ``dy`` with bn3's ReLU sign bits as the GEMM's ``res_mask``; projection
block: the downsample BN backward applies those sign bits to ``dy``, and the downsample dgrad is the residual.
The forward makes the kernel calls of the per-op chain (``ops.bn.conv_bn_act``) and saves the same tensors.
"""
from __future__ import annotations

import torch

from . import bn as _bn
from . import conv as _conv
from . import grad_sink


def _units(block):
    """(conv, bn) pairs in forward order: conv1, conv2, the downsample if any, conv3."""
    ds = [(block.downsample[0], block.downsample[1])] if block.downsample is not None else []
    return [(block.conv1, block.bn1), (block.conv2, block.bn2)] + ds + [(block.conv3, block.bn3)]


def supported(x: torch.Tensor, block) -> bool:
    """NHWC bf16 ``x``; every BN in training mode and on the fused kernels (``ops.bn.module_ok``); conv1 and
    conv3 on the 1x1 GEMM, conv2 and the downsample on the GEMM or the implicit-GEMM kernel (``ops.conv.kind``).
    The activations inside the block are fresh NHWC bf16 tensors like ``x``, so ``x`` stands in for them."""
    if _bn._lib is None or not _bn._nhwc_ok(x):
        return False
    rows1 = x.shape[0] * x.shape[2] * x.shape[3]
    N, _, OH, OW = _bn._out_shape(x, block.conv2)   # conv2, the downsample and conv3 share its output grid
    rows2 = N * OH * OW
    for conv, bn in _units(block):
        if not (bn.training and _bn.module_ok(bn, conv.out_channels, rows1 if conv is block.conv1 else rows2)):
            return False
        k = _conv.kind(x, conv)
        if k != "gemm" and (conv in (block.conv1, block.conv3) or k != "implicit"):
            return False
    return True


def _unit_forward(x, conv, bn, k, relu, residual, need):
    """conv (of kind ``k``) + BN(+residual)(+ReLU); ``need``: whether the conv weight, γ and β need gradients.
    Returns the output and (conv input, weight as the kernel reads it, BN input, ReLU sign bits, mean, invstd, a)."""
    stats = _bn.fused_stats(bn, conv.out_channels, x.device)
    if need[0]:
        grad_sink.note_forward(conv.weight)
    y, w, _ = _conv.forward(x, conv.weight, k, conv.stride[0], conv.padding[0], stats)
    out, mask, ws = _bn.bn_forward(y, bn, residual, relu, stats, need[1:])
    return out, (x, w, y, mask, *ws)


class _BottleneckFn(torch.autograd.Function):
    """Inputs: the block, ``x``, then (conv weight, γ, β) per unit in ``_units`` order."""

    @staticmethod
    def forward(ctx, block, x, *params):
        units = _units(block)
        need = [ctx.needs_input_grad[2 + 3 * i:5 + 3 * i] for i in range(len(units))]
        k = ctx.kinds = [_conv.kind(x, conv) for conv, _ in units]
        h, s1 = _unit_forward(x, *units[0], k[0], True, None, need[0])
        h, s2 = _unit_forward(h, *units[1], k[1], True, None, need[1])
        identity, sd = _unit_forward(x, *units[2], k[2], False, None, need[2]) if len(units) == 4 else (x, ())
        y, s3 = _unit_forward(h, *units[-1], k[-1], True, identity, need[-1])
        ctx.save_for_backward(*s1, *s2, *sd, *s3)
        ctx.block = block
        return y

    @staticmethod
    def backward(ctx, dy):
        units, need = _units(ctx.block), ctx.needs_input_grad
        n = len(units)
        saved = [ctx.saved_tensors[7 * i:7 * i + 7] for i in range(n)]
        grads = [None] * n

        def unit(i, dout, mask, want_dx, residual=None, res_mask=None):
            """BN backward applying ``mask``, then the conv's dgrad (+ ``residual``; GEMM only) and wgrad."""
            (conv, bn), (x, w, y, _, *ws), k = units[i], saved[i], ctx.kinds[i]
            stride, pad = conv.stride[0], conv.padding[0]
            dz, dgamma, dbeta, _ = _bn.bn_backward(dout, bn, y, mask, ws)
            dx = _conv.dgrad(dz, w, k, x.shape, stride, pad, residual, res_mask) if want_dx else None
            dw = _conv.wgrad(dz, x, conv.weight, k, stride, pad) if need[2 + 3 * i] else None
            grads[i] = (dw, dgamma, dbeta)
            return dx

        dy, mask3 = _bn._cl(dy), saved[-1][3]
        d = unit(1, unit(n - 1, dy, mask3, True), saved[1][3], True)
        skip, skip_mask = (unit(2, dy, mask3, need[1]), None) if n == 4 else (dy, mask3)
        dx = unit(0, d, saved[0][3], need[1], skip, skip_mask)
        return (None, dx) + tuple(g for unit_grads in grads for g in unit_grads)


def bottleneck(x: torch.Tensor, block) -> torch.Tensor:
    params = [p for conv, bn in _units(block) for p in (conv.weight, bn.weight, bn.bias)]
    return _BottleneckFn.apply(block, x, *params)
