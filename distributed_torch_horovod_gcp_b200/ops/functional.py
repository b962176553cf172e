"""Functional dispatch layer for the model zoo.

Each function is ONE fusable unit.  ``*_reference`` are plain PyTorch compositions — the CPU
path and the fp32 numerics oracle for the kernels' tests; the CUDA fast paths are the
hand-written sm_90a kernels bound in ``ops.kernels``: wgmma GEMM with fused epilogues
(ops/gemm.py), implicit-GEMM convolution (ops/conv.py), fused BN/ReLU/residual and max-pool
(ops/bn.py), LayerNorm (ops/ln.py), flash attention forward/backward with optional dropout
(ops/attention.py), the LM head fused with its cross-entropy loss (ops/xent.py), dropout fused with the
residual add (ops/dropout.py), the persistent LSTM recurrence (ops/lstm_rec.py) and the LSTM model's linear
head (ops/lstm_fused.py).
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
                residual: Optional[torch.Tensor] = None):
    k = _kernels(x)
    if k is not None and k.has("conv_bn_act"):
        return k.conv_bn_act(x, conv, bn, relu, residual)
    return conv_bn_act_reference(x, conv, bn, relu, residual)


def bottleneck(x, block):
    """ResNet bottleneck block (``models.resnet.Bottleneck``).  Kernel path: one autograd node whose
    backward adds the skip-connection gradient in conv1's dgrad epilogue (ops/bottleneck.py).  Otherwise
    (CPU, eval mode, shapes that node does not cover) the per-op chain, where autograd adds it."""
    k = _kernels(x)
    if k is not None and k.has("conv_bn_act"):
        from . import bottleneck as _bt
        if _bt.supported(x, block):
            return _bt.bottleneck(x, block)
    out = conv_bn_act(x, block.conv1, block.bn1, relu=True)
    out = conv_bn_act(out, block.conv2, block.bn2, relu=True)
    identity = x if block.downsample is None else \
        conv_bn_act(x, block.downsample[0], block.downsample[1], relu=False)
    return conv_bn_act(out, block.conv3, block.bn3, relu=True, residual=identity)


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
    if k is not None and k.has("linear") and k.linear_supported(x, weight, bias, residual):
        return k.linear(x, weight, bias, act, residual)
    return linear_reference(x, weight, bias, act, residual)


def mlp(x, w1, b1, w2, b2, residual=None):
    """Transformer MLP: fc2(gelu(fc1(x))) + residual (one fused autograd node on the kernel path)."""
    k = _kernels(x)
    if k is not None and k.has("linear") and b1 is not None and b2 is not None \
            and k.linear_supported(x, w1, b1, residual, w2=w2, b2=b2):
        return k.mlp(x, w1, b1, w2, b2, residual)
    return linear_reference(linear_reference(x, w1, b1, act="gelu"), w2, b2, residual=residual)


# ------------------------------------------------------------------ dropout (+ residual)
def _check_p(p) -> float:
    p = float(p)
    if not 0.0 <= p <= 1.0:
        raise ValueError(f"dropout probability must be in [0, 1], got {p}")
    return p


def dropout_add_reference(y, residual, p: float):
    y = F.dropout(y, p)
    return y if residual is None else residual + y


def dropout_add(y, residual, p: float):
    """``residual + F.dropout(y, p)`` (training-mode dropout; ``residual=None``: ``F.dropout(y, p)``).  Kernel
    path (contiguous bf16 ``y`` and ``residual`` of one shape, numel % 8 == 0): one pass that draws the keep
    mask, scales and adds (ops/dropout.py); its backward draws the same mask again from the saved seed.
    ``p == 0`` adds ``y`` as it is.  Anything else takes the composition above."""
    p = _check_p(p)
    if p == 0.0:
        return y if residual is None else residual + y
    k = _kernels(y)
    if k is not None and k.has("dropout_add") and k.dropout_add_supported(y, residual):
        return k.dropout_add(y, residual, p)
    return dropout_add_reference(y, residual, p)


# ------------------------------------------------------------------ layer norm
def layer_norm(x, weight, bias, eps: float = 1e-6):
    k = _kernels(x)
    if k is not None and k.has("layer_norm") and k.layer_norm_supported(x, weight, bias):
        return k.layer_norm(x, weight, bias, eps)
    return F.layer_norm(x, (x.shape[-1],), None if weight is None else weight.to(x.dtype),
                        None if bias is None else bias.to(x.dtype), eps)


# ------------------------------------------------------------------ attention
def attention_reference(qkv, heads: int, causal: bool = False, dropout_p: float = 0.0):
    """Self-attention of a packed ``[B, S, 3 D]`` q|k|v tensor; ``causal=True``: position i attends to
    positions 0..i only; ``dropout_p``: dropout on the attention probabilities."""
    dropout_p = _check_p(dropout_p)
    B, S, D3 = qkv.shape
    D = D3 // 3
    hd = D // heads
    q, k, v = qkv.view(B, S, 3, heads, hd).permute(2, 0, 3, 1, 4)
    o = F.scaled_dot_product_attention(q, k, v, dropout_p=dropout_p, is_causal=causal)
    return o.transpose(1, 2).reshape(B, S, D)


def attention(qkv, heads: int, causal: bool = False, dropout_p: float = 0.0):
    """Self-attention of a packed ``[B, S, 3 D]`` tensor: always the SDPA composition.  The flash-attention
    kernels take q, k and v as the three dense projection outputs ``qkv_attention`` makes."""
    return attention_reference(qkv, heads, causal, dropout_p)


def qkv_attention(x, weight, bias, heads: int, causal: bool = False, dropout_p: float = 0.0,
                  sequence_parallel: bool = False, process_set=None):
    """Multi-head self-attention input stage: packed QKV projection + scaled-dot-product attention
    (``causal=True``: position i attends to positions 0..i only, as in a decoder; ``dropout_p``: dropout on
    the attention probabilities, drawn inside the flash-attention kernels on the kernel path).
    Kernel path: q, k, v are produced as three dense matrices (no un-pack / re-pack copies).
    ``sequence_parallel=True``: ``x`` is this rank's zigzag shard of the sequence and attention runs through
    ``seq_parallel.sp_attention`` over every rank's keys and values (``process_set``: the ranks of that set
    only)."""
    dropout_p = _check_p(dropout_p)
    if sequence_parallel:
        return _sp_qkv_attention(x, weight, bias, heads, causal, dropout_p, process_set)
    k = _kernels(x)
    if k is not None and k.has("linear") and k.linear_supported(x, weight, bias) and x.dim() == 3 \
            and weight.shape[0] == 3 * x.shape[-1] and weight.shape[0] % 24 == 0 and x.shape[-1] % heads == 0 \
            and os.environ.get("B200DP_SPLIT_QKV", "1") == "1":
        B, S, D = x.shape
        hd = D // heads
        q, kk, v = k.qkv_proj(x, weight, bias)
        q, kk, v = [t.view(B, S, heads, hd).transpose(1, 2) for t in (q, kk, v)]
        if k.has("attention_fused") and hd == 64 and os.environ.get("B200DP_ATTN_KERNEL", "1") == "1":
            from . import attention as _attn
            if _attn.supported(q, kk, v):
                o = _attn.attention_fused(q, kk, v, causal, dropout_p)   # [B,H,S,hd] view of [B,S,H,hd] memory
                return o.transpose(1, 2).reshape(B, S, D)  # a view: no copy
        o = F.scaled_dot_product_attention(q, kk, v, dropout_p=dropout_p, is_causal=causal)
        return o.transpose(1, 2).reshape(B, S, D)
    return attention(linear(x, weight, bias), heads, causal, dropout_p)


def _sp_qkv_attention(x, weight, bias, heads, causal, dropout_p, process_set=None):
    from .seq_parallel import sp_attention
    B, S, D = x.shape
    hd = D // heads
    k = _kernels(x)
    if k is not None and k.has("linear") and k.linear_supported(x, weight, bias) and weight.shape[0] == 3 * D \
            and weight.shape[0] % 24 == 0 and D % heads == 0:
        q, kk, v = [t.view(B, S, heads, hd).transpose(1, 2) for t in k.qkv_proj(x, weight, bias)]
    else:
        q, kk, v = linear(x, weight, bias).view(B, S, 3, heads, hd).permute(2, 0, 3, 1, 4)
    return sp_attention(q, kk, v, causal, dropout_p, process_set).transpose(1, 2).reshape(B, S, D)


# ------------------------------------------------------------------ LM head + cross-entropy
def linear_cross_entropy_reference(x, weight, targets, ignore_index: int = -100, reduction: str = "mean"):
    logits = F.linear(x, weight).float()
    return F.cross_entropy(logits.reshape(-1, logits.shape[-1]), targets.reshape(-1), ignore_index=ignore_index,
                           reduction=reduction)


def linear_cross_entropy(x, weight, targets, ignore_index: int = -100, reduction: str = "mean"):
    """``F.cross_entropy(F.linear(x, weight).float(), targets.reshape(-1), ignore_index, reduction)`` for
    ``x`` [..., D], ``weight`` [V, D] and int64 ``targets`` with ``x.shape[:-1]`` elements; ``"none"`` returns
    fp32 [N], ``"sum"`` / ``"mean"`` an fp32 scalar.

    Kernel path (bf16 ``x`` and ``weight`` on an sm_90 device, D % 8 == 0, V % 8 == 0, 16-byte-aligned
    rows): the [N, V] logits are never stored (ops/xent.py); the backward holds one bf16 chunk of at most
    256 MiB of them.  There, a target outside [0, V) that is not ``ignore_index`` gives its row a NaN loss
    and a NaN gradient row instead of torch's device assert.  Anything else takes the composition above."""
    if reduction not in ("none", "sum", "mean"):
        raise ValueError(f"reduction must be 'none', 'sum' or 'mean'; got {reduction!r}")
    if weight.dim() != 2 or x.dim() < 1 or x.shape[-1] != weight.shape[1]:
        raise ValueError(f"x [..., D] and weight [V, D] do not match: {tuple(x.shape)} and {tuple(weight.shape)}")
    n_rows = x.numel() // x.shape[-1] if x.shape[-1] else 0
    if targets.numel() != n_rows:
        raise ValueError(f"targets has {targets.numel()} elements; x has {n_rows} rows")
    k = _kernels(x)
    if k is not None and k.has("linear_cross_entropy") and k.linear_cross_entropy_supported(x, weight, targets):
        return k.linear_cross_entropy(x, weight, targets, ignore_index, reduction)
    return linear_cross_entropy_reference(x, weight, targets, ignore_index, reduction)


# ------------------------------------------------------------------ LSTM recurrence and head
def lstm_reference(x, module: nn.LSTM, hidden):
    return module(x, hidden)


_warned_cudnn = False


def lstm(x, module: nn.LSTM, hidden):
    """``module(x, hidden) -> (seq, (h_n, c_n))``.  Kernel path (hidden size 256, fp32, batch_first, biases,
    1..512 input features, no projection): the persistent recurrence kernels for the whole stack, inter-layer
    dropout included (ops/lstm_rec.py).  Any other LSTM takes cuDNN's RNN, logged once when it could have
    taken the kernels but for its shape or dtype."""
    k = _kernels(x)
    if k is not None and k.has("lstm_recurrent"):
        from . import lstm_rec
        if lstm_rec.stack_supported(module, x):
            return lstm_rec.lstm_stack(x, hidden[0], hidden[1], [w for ws in module.all_weights for w in ws],
                                       module.num_layers, module.bidirectional,
                                       dropout=module.dropout if module.training else 0.0)
        global _warned_cudnn
        if not _warned_cudnn:
            _warned_cudnn = True
            import logging
            logging.getLogger("b200dp").warning(
                "LSTM shape (layers=%d, hidden=%d, features=%d, bidirectional=%s, proj_size=%d, dtype=%s) is "
                "outside the persistent recurrence kernels (hidden size 256, 1..512 features, fp32, no "
                "projection): using the cuDNN RNN for this module",
                module.num_layers, module.hidden_size, module.input_size, module.bidirectional,
                module.proj_size, module.weight_hh_l0.dtype)
    return lstm_reference(x, module, hidden)


def lstm_head_reference(seq, t: int, l1: nn.Linear, l2: nn.Linear, l3: nn.Linear):
    return l3(l2(l1(seq[:, t:t + 1])))


def lstm_head(seq, t: int, l1: nn.Linear, l2: nn.Linear, l3: nn.Linear):
    """``l3(l2(l1(seq[:, t:t + 1])))``, ``[B, 1, out3]``.  Kernel path (fp32, batch <= 1024, in + out1 + out2 +
    out3 <= 12000, the six linear tensors dense fp32 on ``seq``'s device): the step gather and the three
    linears as one forward and two backward kernels (ops/lstm_fused.py)."""
    k = _kernels(seq)
    if k is not None and k.has("lstm_fused") and k.lstm_head_supported(seq, t, l1, l2, l3):
        return k.lstm_head(seq, t, l1, l2, l3)
    return lstm_head_reference(seq, t, l1, l2, l3)


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
