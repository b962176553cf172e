"""Flash attention binding (csrc/attn_sm90.cu): wgmma forward + backward, bf16, head dim 64,
non-causal (the ViT-B/16 configuration).  ``attention_fused(q, k, v)`` takes ``[B, H, S, 64]``
tensors with ANY batch/head/sequence strides (64 contiguous) — in the model they are the three dense
``[B*S, D]`` projection outputs viewed as ``[B, S, H, 64]`` and transposed, so no un-pack / re-pack
copy exists in either direction: the output and all three gradients are produced in ``[B, S, H, 64]``
memory order, i.e. directly as the ``[B*S, D]`` matrices the neighbouring GEMMs consume.
Replaces ``F.scaled_dot_product_attention`` (cuDNN / flash library kernels)."""
from __future__ import annotations

import ctypes
import math

import torch

from . import counters

_lib = None


def register(lib, have):
    global _lib
    if not hasattr(lib, "b200dp_attn_fwd"):
        return
    _lib = lib
    vp, i, f, u64 = ctypes.c_void_p, ctypes.c_int, ctypes.c_float, ctypes.c_uint64
    lp = ctypes.POINTER(ctypes.c_longlong)
    lib.b200dp_attn_fwd.argtypes = [vp, vp, vp, vp, vp, i, i, i, i, lp, lp, lp, lp, f, u64]
    lib.b200dp_attn_bwd.argtypes = [vp] * 10 + [i, i, i, i] + [lp] * 8 + [f, u64]
    lib.b200dp_attn_last_error.restype = ctypes.c_char_p
    if hasattr(lib, "b200dp_cast_acc_zero"):
        lib.b200dp_cast_acc_zero.argtypes = [vp, vp, ctypes.c_longlong, i, i, i, u64]
    have["attention_fused"] = True


def _ck(rc):
    if rc != 0:
        raise RuntimeError("attention kernel: " + (_lib.b200dp_attn_last_error() or b"").decode())


def _strides(t):
    """(batch, head, seq) element strides of a [B, H, S, D] tensor."""
    return (ctypes.c_longlong * 3)(t.stride(0), t.stride(1), t.stride(2))


def _ok(t: torch.Tensor) -> bool:
    return (t.dtype == torch.bfloat16 and t.dim() == 4 and t.shape[3] == 64 and t.stride(3) == 1
            and t.data_ptr() % 16 == 0 and all(s % 8 == 0 for s in t.stride()[:3]))


def supported(q, k, v) -> bool:
    return _lib is not None and q.is_cuda and _ok(q) and _ok(k) and _ok(v) and q.shape == k.shape == v.shape


def _fix(t):
    return t if _ok(t) else t.contiguous()


_ws = {}


def _dq_workspace(B, S, H, dev):
    key = (B, S, H, dev.index)
    w = _ws.get(key)
    if w is None:
        w = torch.zeros((B, S, H, 64), dtype=torch.float32, device=dev)
        _ws[key] = w
    return w


class _AttnFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, q, k, v):
        q, k, v = _fix(q), _fix(k), _fix(v)
        B, H, S, D = q.shape
        dev = q.device
        o = torch.empty((B, S, H, D), dtype=torch.bfloat16, device=dev).permute(0, 2, 1, 3)
        need = any(ctx.needs_input_grad)
        lse = torch.empty((B, H, S), dtype=torch.float32, device=dev) if need else None
        scale = 1.0 / math.sqrt(D)
        _ck(_lib.b200dp_attn_fwd(q.data_ptr(), k.data_ptr(), v.data_ptr(), o.data_ptr(),
                                 lse.data_ptr() if lse is not None else None, B, H, S, D,
                                 _strides(q), _strides(k), _strides(v), _strides(o), scale,
                                 torch.cuda.current_stream(dev).cuda_stream))
        counters.bump("attn_fwd")
        if need:
            ctx.save_for_backward(q, k, v, o, lse)
        return o

    @staticmethod
    def backward(ctx, do):
        q, k, v, o, lse = ctx.saved_tensors
        B, H, S, D = q.shape
        dev = q.device
        do = _fix(do)
        acc = _dq_workspace(B, S, H, dev)                       # [B, S, H, 64] fp32, zero on entry
        acc_v = acc.permute(0, 2, 1, 3)
        delta = torch.empty((B, H, S), dtype=torch.float32, device=dev)
        dq, dk, dv = [torch.empty((B, S, H, D), dtype=torch.bfloat16, device=dev).permute(0, 2, 1, 3)
                      for _ in range(3)]
        st = torch.cuda.current_stream(dev).cuda_stream
        _ck(_lib.b200dp_attn_bwd(q.data_ptr(), k.data_ptr(), v.data_ptr(), o.data_ptr(), do.data_ptr(),
                                 lse.data_ptr(), delta.data_ptr(), acc.data_ptr(), dk.data_ptr(), dv.data_ptr(),
                                 B, H, S, D, _strides(q), _strides(k), _strides(v), _strides(o), _strides(do),
                                 _strides(acc_v), _strides(dk), _strides(dv), 1.0 / math.sqrt(D), st))
        rc = _lib.b200dp_cast_acc_zero(acc.data_ptr(), dq.data_ptr(), acc.numel(), 1, 0, 1, st)
        if rc != 0:
            raise RuntimeError("cast_acc_zero failed")
        counters.bump("attn_bwd", 3)
        return dq, dk, dv


def attention_fused(q, k, v):
    """softmax(q k^T / sqrt(64)) v for [B, H, S, 64] bf16 tensors; returns [B, H, S, 64] (memory order
    [B, S, H, 64])."""
    return _AttnFn.apply(q, k, v)
