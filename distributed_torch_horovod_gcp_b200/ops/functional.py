"""Functional dispatch layer for the model zoo.

Each function is ONE fusable unit.  ``*_reference`` are plain PyTorch compositions — the CPU
path and the fp32 numerics oracle for the kernels' tests; the CUDA fast paths are the
hand-written sm_90a kernels bound in ``ops.kernels``: wgmma GEMM with fused epilogues
(ops/gemm.py), implicit-GEMM convolution (ops/conv.py), fused BN/ReLU/residual and max-pool
(ops/bn.py), LayerNorm (ops/ln.py), flash attention forward/backward (ops/attention.py).
"""
from __future__ import annotations

import os
from typing import Optional

import torch
import torch.nn.functional as F
from torch import nn

_FORCE_REFERENCE = os.environ.get("B200DP_REFERENCE_OPS", "0") == "1"


def _kernels(x: torch.Tensor):
    """Return the kernels module when ``x`` can take the sm_90a path, else ``None``."""
    if _FORCE_REFERENCE or not x.is_cuda:
        return None
    from . import kernels
    return kernels if kernels.enabled_for(x) else None


# ------------------------------------------------------------------ conv + BN (+ReLU, +residual)
def conv_bn_act_reference(x, conv: nn.Conv2d, bn: nn.BatchNorm2d, relu: bool,
                          residual: Optional[torch.Tensor] = None):
    y = F.conv2d(x, conv.weight.to(x.dtype), None, conv.stride, conv.padding)
    y = bn(y)
    if residual is not None:
        y = y + residual
    return F.relu(y) if relu else y


def conv_bn_act(x, conv: nn.Conv2d, bn: nn.BatchNorm2d, relu: bool = True,
                residual: Optional[torch.Tensor] = None, skip_box=None, input_box=None, park_box=None):
    """``skip_box`` / ``input_box`` (kernel path only): see ``ops.grad_sink.GradBox`` — the block's last
    BN parks the skip-connection gradient, the block's first conv adds it in its dgrad epilogue."""
    k = _kernels(x)
    if k is not None and k.has("conv_bn_act"):
        return k.conv_bn_act(x, conv, bn, relu, residual, skip_box=skip_box, input_box=input_box,
                             park_box=park_box)
    return conv_bn_act_reference(x, conv, bn, relu, residual)


def new_grad_box(x: torch.Tensor):
    """A GradBox when ``x`` takes the kernel path and needs a gradient, else ``None``."""
    if _kernels(x) is None or not x.requires_grad or not torch.is_grad_enabled():
        return None
    from .grad_sink import GradBox
    return GradBox()


def max_pool_3x3_s2(x):
    k = _kernels(x)
    if k is not None and k.has("max_pool_3x3_s2"):
        return k.max_pool_3x3_s2(x)
    return F.max_pool2d(x, kernel_size=3, stride=2, padding=1)


def global_avg_pool(x):
    k = _kernels(x)
    if k is not None and k.has("global_avg_pool"):
        return k.global_avg_pool(x)
    return x.mean(dim=(2, 3))


# ------------------------------------------------------------------ linear (+bias, +act, +residual)
def linear_reference(x, weight, bias=None, act: Optional[str] = None, residual=None):
    y = F.linear(x, weight.to(x.dtype), None if bias is None else bias.to(x.dtype))
    if act == "gelu":
        y = F.gelu(y)
    elif act == "relu":
        y = F.relu(y)
    if residual is not None:
        y = y + residual
    return y


def linear(x, weight, bias=None, act: Optional[str] = None, residual=None):
    k = _kernels(x)
    if k is not None and k.has("linear") and k.linear_supported(x, weight):
        return k.linear(x, weight, bias, act, residual)
    return linear_reference(x, weight, bias, act, residual)


def mlp(x, w1, b1, w2, b2, residual=None):
    """Transformer MLP: fc2(gelu(fc1(x))) + residual (one fused autograd node on the kernel path)."""
    k = _kernels(x)
    if k is not None and k.has("linear") and k.linear_supported(x, w1) and b1 is not None \
            and b2 is not None and w2.shape[0] % 8 == 0:
        return k.mlp(x, w1, b1, w2, b2, residual)
    return linear_reference(linear_reference(x, w1, b1, act="gelu"), w2, b2, residual=residual)


# ------------------------------------------------------------------ layer norm
def layer_norm(x, weight, bias, eps: float = 1e-6):
    k = _kernels(x)
    if k is not None and k.has("layer_norm") and k.layer_norm_supported(x, weight):
        return k.layer_norm(x, weight, bias, eps)
    return F.layer_norm(x, (x.shape[-1],), weight.to(x.dtype), bias.to(x.dtype), eps)


# ------------------------------------------------------------------ attention
def attention_reference(qkv, heads: int):
    B, S, D3 = qkv.shape
    D = D3 // 3
    hd = D // heads
    q, k, v = qkv.view(B, S, 3, heads, hd).permute(2, 0, 3, 1, 4)
    o = F.scaled_dot_product_attention(q, k, v)
    return o.transpose(1, 2).reshape(B, S, D)


def attention(qkv, heads: int):
    k = _kernels(qkv)
    if k is not None and k.has("attention"):
        return k.attention(qkv, heads)
    return attention_reference(qkv, heads)


def qkv_attention(x, weight, bias, heads: int):
    """Multi-head self-attention input stage: packed QKV projection + scaled-dot-product attention.
    Kernel path: q, k, v are produced as three dense matrices (no un-pack / re-pack copies)."""
    k = _kernels(x)
    if k is not None and k.has("linear") and k.linear_supported(x, weight) and weight.shape[0] % 24 == 0 \
            and os.environ.get("B200DP_SPLIT_QKV", "1") == "1":
        B, S, D = x.shape
        hd = D // heads
        q, kk, v = k.qkv_proj(x, weight, bias)
        q, kk, v = [t.view(B, S, heads, hd).transpose(1, 2) for t in (q, kk, v)]
        if k.has("attention_fused") and hd == 64 and os.environ.get("B200DP_ATTN_KERNEL", "1") == "1":
            from . import attention as _attn
            if _attn.supported(q, kk, v):
                o = _attn.attention_fused(q, kk, v)       # [B,H,S,hd] view of [B,S,H,hd] memory
                return o.transpose(1, 2).reshape(B, S, D)  # a view: no copy
        o = F.scaled_dot_product_attention(q, kk, v)
        return o.transpose(1, 2).reshape(B, S, D)
    return attention(linear(x, weight, bias), heads)


# ------------------------------------------------------------------ ViT patch embedding
def patch_embed(x, weight, bias, patch: int):
    """``[B,3,H,W]`` (NCHW logical, any memory format) -> ``[B, (H/p)*(W/p), D]``: gather
    non-overlapping patches to rows and run ONE GEMM against ``weight`` viewed as
    ``[D, 3*p*p]`` (identical to the stride-p conv, but GEMM-shaped for the wgmma GEMM)."""
    B, C, H, W = x.shape
    gh, gw = H // patch, W // patch
    cols = x.reshape(B, C, gh, patch, gw, patch).permute(0, 2, 4, 1, 3, 5) \
            .reshape(B, gh * gw, C * patch * patch)
    return linear(cols, weight.reshape(weight.shape[0], -1), bias)
