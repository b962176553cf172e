"""Gradient compression (wire dtype) — Horovod's ``hvd.Compression`` shape (SURVEY.md §2.3;
default ``none`` at the reference's call site app/torch_train.py:259).

On H100 the interesting setting is ``bf16``: gradients travel NVLink as bf16 and are
accumulated in fp32 registers inside the fused allreduce kernel, which halves link bytes.
"""
from __future__ import annotations

import torch


class Compressor:
    @staticmethod
    def compress(tensor):
        raise NotImplementedError

    @staticmethod
    def decompress(tensor, ctx):
        raise NotImplementedError


class NoneCompressor(Compressor):
    wire_dtype = None

    @staticmethod
    def compress(tensor):
        return tensor, None

    @staticmethod
    def decompress(tensor, ctx):
        return tensor


class _CastCompressor(Compressor):
    wire_dtype = torch.float16

    @classmethod
    def compress(cls, tensor):
        if tensor.dtype.is_floating_point and tensor.dtype != cls.wire_dtype:
            return tensor.to(cls.wire_dtype), tensor.dtype
        return tensor, None

    @staticmethod
    def decompress(tensor, ctx):
        return tensor.to(ctx) if ctx is not None else tensor


class FP16Compressor(_CastCompressor):
    wire_dtype = torch.float16


class BF16Compressor(_CastCompressor):
    wire_dtype = torch.bfloat16


class Compression:
    none = NoneCompressor
    fp16 = FP16Compressor
    bf16 = BF16Compressor
