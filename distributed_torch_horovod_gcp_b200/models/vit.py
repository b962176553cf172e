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
    def __init__(self, dim: int, heads: int, mlp_dim: int):
        super().__init__()
        self.heads = heads
        self.ln_1 = nn.LayerNorm(dim, eps=1e-6)
        self.qkv = nn.Linear(dim, 3 * dim)
        self.proj = nn.Linear(dim, dim)
        self.ln_2 = nn.LayerNorm(dim, eps=1e-6)
        self.fc1 = nn.Linear(dim, mlp_dim)
        self.fc2 = nn.Linear(mlp_dim, dim)

    def forward(self, x):
        B, S, D = x.shape
        h = F2.layer_norm(x, self.ln_1.weight, self.ln_1.bias, self.ln_1.eps)
        a = F2.qkv_attention(h, self.qkv.weight, self.qkv.bias, self.heads)   # [B,S,D]
        x = F2.linear(a, self.proj.weight, self.proj.bias, residual=x)
        h = F2.layer_norm(x, self.ln_2.weight, self.ln_2.bias, self.ln_2.eps)
        return F2.mlp(h, self.fc1.weight, self.fc1.bias, self.fc2.weight, self.fc2.bias, residual=x)


class VisionTransformer(nn.Module):
    def __init__(self, image_size=224, patch=16, dim=768, depth=12, heads=12, mlp_dim=3072,
                 num_classes=1000):
        super().__init__()
        self.patch, self.dim = patch, dim
        n = (image_size // patch) ** 2
        self.conv_proj = nn.Conv2d(3, dim, patch, stride=patch)
        self.class_token = nn.Parameter(torch.zeros(1, 1, dim))
        self.pos_embedding = nn.Parameter(torch.empty(1, n + 1, dim).normal_(std=0.02))
        self.layers = nn.ModuleList([EncoderBlock(dim, heads, mlp_dim) for _ in range(depth)])
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
