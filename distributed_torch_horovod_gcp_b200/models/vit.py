"""Vision Transformer ViT-B/16 ([DRIVER] BASELINE.json config 4, "GEMM-bound path"; not in
the reference — SURVEY.md §0 item 6).  86 567 656 parameters in 152 tensors at 224x224 /
1000 classes, matching the survey's count.

Every matmul goes through ``ops.functional.linear`` (wgmma GEMM with fused bias / GELU /
residual epilogues when the in-tree kernels are built) and attention through
``ops.functional.attention``; the patch embedding is a stride-16 16x16 convolution, i.e. a
pure ``[N*196, 768] x [768, 768]`` GEMM after an NHWC patch gather.
"""
from __future__ import annotations

import torch
from torch import nn

from ..ops import functional as F2


class EncoderBlock(nn.Module):
    """Pre-LN transformer block.  ``causal=True`` makes it a decoder block (``models.gpt``).

    In training mode, ``attention_dropout`` drops attention probabilities (inside the flash-attention kernels)
    and ``dropout`` drops the output of each residual branch (after ``proj`` and after ``fc2``) before it is
    added to the stream.  With both at 0, or in eval mode, the block computes what it computes without them."""

    def __init__(self, dim: int, heads: int, mlp_dim: int, causal: bool = False, eps: float = 1e-6,
                 dropout: float = 0.0, attention_dropout: float = 0.0):
        super().__init__()
        for name, p in (("dropout", dropout), ("attention_dropout", attention_dropout)):
            if not 0.0 <= p <= 1.0:
                raise ValueError(f"{name} must be in [0, 1], got {p}")
        self.heads = heads
        self.causal = causal
        self.dropout, self.attention_dropout = float(dropout), float(attention_dropout)
        self.ln_1 = nn.LayerNorm(dim, eps=eps)
        self.qkv = nn.Linear(dim, 3 * dim)
        self.proj = nn.Linear(dim, dim)
        self.ln_2 = nn.LayerNorm(dim, eps=eps)
        self.fc1 = nn.Linear(dim, mlp_dim)
        self.fc2 = nn.Linear(mlp_dim, dim)

    def forward(self, x, sequence_parallel: bool = False, process_set=None):
        """``sequence_parallel=True``: ``x`` is this rank's zigzag shard of the sequence (``ops.seq_parallel``),
        split across the ranks of ``process_set`` (an ``hvd.ProcessSet``; None: the world)."""
        B, S, D = x.shape
        pa = self.attention_dropout if self.training else 0.0
        pr = self.dropout if self.training else 0.0
        h = F2.layer_norm(x, self.ln_1.weight, self.ln_1.bias, self.ln_1.eps)
        a = F2.qkv_attention(h, self.qkv.weight, self.qkv.bias, self.heads, self.causal, pa,
                             sequence_parallel=sequence_parallel, process_set=process_set)   # [B,S,D]
        if pr > 0.0:
            # the branch output is dropped before the add, so the GEMM epilogue adds no residual
            x = F2.dropout_add(F2.linear(a, self.proj.weight, self.proj.bias), x, pr)
            h = F2.layer_norm(x, self.ln_2.weight, self.ln_2.bias, self.ln_2.eps)
            return F2.dropout_add(F2.mlp(h, self.fc1.weight, self.fc1.bias, self.fc2.weight, self.fc2.bias), x, pr)
        x = F2.linear(a, self.proj.weight, self.proj.bias, residual=x)
        h = F2.layer_norm(x, self.ln_2.weight, self.ln_2.bias, self.ln_2.eps)
        return F2.mlp(h, self.fc1.weight, self.fc1.bias, self.fc2.weight, self.fc2.bias, residual=x)


class VisionTransformer(nn.Module):
    """ViT with torchvision's ``vit_b_16`` structure.  ``dropout`` drops, in training mode, the tokens after
    the position embedding is added and the output of each block's two residual branches;
    ``attention_dropout`` drops attention probabilities.  Unlike torchvision, nothing is dropped between the
    MLP's GELU and ``fc2``: that point is inside the fused MLP node."""

    def __init__(self, image_size=224, patch=16, dim=768, depth=12, heads=12, mlp_dim=3072,
                 num_classes=1000, dropout: float = 0.0, attention_dropout: float = 0.0):
        super().__init__()
        if not 0.0 <= dropout <= 1.0:
            raise ValueError(f"dropout must be in [0, 1], got {dropout}")
        self.patch, self.dim = patch, dim
        self.dropout = float(dropout)
        n = (image_size // patch) ** 2
        self.conv_proj = nn.Conv2d(3, dim, patch, stride=patch)
        self.class_token = nn.Parameter(torch.zeros(1, 1, dim))
        self.pos_embedding = nn.Parameter(torch.empty(1, n + 1, dim).normal_(std=0.02))
        self.layers = nn.ModuleList([EncoderBlock(dim, heads, mlp_dim, dropout=dropout,
                                                  attention_dropout=attention_dropout) for _ in range(depth)])
        self.ln = nn.LayerNorm(dim, eps=1e-6)
        self.head = nn.Linear(dim, num_classes)
        nn.init.trunc_normal_(self.conv_proj.weight, std=(1.0 / (3 * patch * patch)) ** 0.5)
        nn.init.zeros_(self.conv_proj.bias)
        nn.init.zeros_(self.head.weight)
        nn.init.zeros_(self.head.bias)

    def forward(self, x):
        B = x.shape[0]
        x = F2.patch_embed(x, self.conv_proj.weight, self.conv_proj.bias, self.patch)  # [B,n,D]
        x = torch.cat([self.class_token.expand(B, -1, -1).to(x.dtype), x], dim=1)
        x = x + self.pos_embedding.to(x.dtype)
        if self.training and self.dropout > 0.0:
            x = F2.dropout_add(x, None, self.dropout)
        for blk in self.layers:
            x = blk(x)
        x = F2.layer_norm(x[:, 0], self.ln.weight, self.ln.bias, self.ln.eps)
        return F2.linear(x, self.head.weight, self.head.bias)


def vit_b_16(**kw):
    return VisionTransformer(**kw)


def vit_tiny(**kw):
    d = dict(image_size=32, patch=8, dim=64, depth=2, heads=4, mlp_dim=128, num_classes=10)
    d.update(kw)
    return VisionTransformer(**d)
