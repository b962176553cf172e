"""Fused LM-head cross-entropy binding (csrc/xent_sm90.cu) and its autograd node.

    loss = cross_entropy(x @ W^T, targets)     x [N, D], W [V, D] bf16, targets [N] int64

Forward: ``xent_fwd_kernel`` computes each logit tile in wgmma registers and keeps only a running
(max, sum of exp) per row; a finish kernel folds those into ``lse`` [N] and the loss.  No [N, V] tensor is
allocated.  Backward, in row chunks of at most ``_CHUNK_BYTES`` of bf16 dlogits:
  dlogits = s_i (softmax(x W^T) - onehot(t))   xent_grad_kernel recomputes the chunk's logit tiles
  dX rows = dlogits @ W                         gemm, W MN-major (as gemm.dgrad)
  dW     += dlogits^T @ x rows                  gemm, both MN-major (as gemm.wgrad); fp32 across chunks
Every sum runs in a fixed order, so two runs give the same bits, and nothing is read back to the host.
"""
from __future__ import annotations

import ctypes

import torch

from . import counters
from . import gemm as _gemm
from . import grad_sink

_lib = None
# bytes of one chunk of bf16 dlogits in the backward (at V = 50304: 2560 rows, 258 MB)
_CHUNK_BYTES = 256 << 20
REDUCTIONS = ("none", "sum", "mean")


def register(lib, have):
    global _lib
    if not hasattr(lib, "b200dp_xent_fwd"):
        return
    _lib = lib
    vp, i, ll, u64 = ctypes.c_void_p, ctypes.c_int, ctypes.c_longlong, ctypes.c_uint64
    lib.b200dp_xent_fwd.argtypes = [vp, vp, vp, vp, vp, vp, vp, i, i, i, ll, i, i, u64]
    lib.b200dp_xent_fwd.restype = i
    lib.b200dp_xent_grad.argtypes = [vp, vp, vp, vp, vp, i, vp, vp, i, i, i, i, i, ll, i, u64]
    lib.b200dp_xent_grad.restype = i
    lib.b200dp_xent_last_error.restype = ctypes.c_char_p
    have["linear_cross_entropy"] = True


def _ck(rc, what):
    if rc != 0:
        raise RuntimeError(f"{what}: " + (_lib.b200dp_xent_last_error() or b"").decode())


def supported(x: torch.Tensor, weight: torch.Tensor, targets: torch.Tensor) -> bool:
    if _lib is None or x.dtype != torch.bfloat16 or weight.dtype != torch.bfloat16:
        return False
    if weight.dim() != 2 or targets.dtype != torch.int64 or targets.device != x.device or weight.device != x.device:
        return False
    V, D = weight.shape
    N = x.numel() // max(D, 1)
    return (D % 8 == 0 and V % 8 == 0 and 0 < N < (1 << 24) and weight.stride(1) == 1 and weight.stride(0) == D
            and weight.data_ptr() % 16 == 0)


def chunk_rows(V: int) -> int:
    """Rows of one backward chunk: a multiple of 128 whose bf16 [rows, V] dlogits fit in ``_CHUNK_BYTES``."""
    return max(128, (_CHUNK_BYTES // (2 * V)) // 128 * 128)


def _rows(t: torch.Tensor, D: int) -> torch.Tensor:
    t2 = t.reshape(-1, D)
    if t2.stride(-1) != 1 or t2.stride(0) != D or t2.data_ptr() % 16:
        t2 = t2.contiguous()
    return t2


class _LinearXentFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, weight, targets, ignore_index, reduction, max_ctas):
        V, D = weight.shape
        x2 = _rows(x, D)
        t = targets.reshape(-1).contiguous()
        N = x2.shape[0]
        dev = x.device
        if ctx.needs_input_grad[1]:
            grad_sink.note_forward(weight)
        lse = torch.empty(N, dtype=torch.float32, device=dev)
        rows = torch.empty(N, dtype=torch.float32, device=dev) if reduction == "none" else None
        stats = torch.empty(2, dtype=torch.float32, device=dev) if reduction != "none" else None
        out = torch.empty((), dtype=torch.float32, device=dev) if reduction != "none" else None
        _ck(_lib.b200dp_xent_fwd(x2.data_ptr(), weight.data_ptr(), t.data_ptr(), lse.data_ptr(),
                                 rows.data_ptr() if rows is not None else None,
                                 stats.data_ptr() if stats is not None else None,
                                 out.data_ptr() if out is not None else None, N, D, V, int(ignore_index),
                                 int(reduction == "mean"), int(max_ctas),
                                 torch.cuda.current_stream(dev).cuda_stream), "b200dp_xent_fwd")
        counters.bump("xent_fwd", 2 if stats is None else 3)
        ctx.save_for_backward(x2, weight, t, lse, stats)
        ctx.x_shape, ctx.ignore_index, ctx.reduction, ctx.max_ctas = x.shape, int(ignore_index), reduction, max_ctas
        return rows if rows is not None else out

    @staticmethod
    def backward(ctx, g):
        x2, weight, t, lse, stats = ctx.saved_tensors
        V, D = weight.shape
        N = x2.shape[0]
        dev = x2.device
        need_dx, need_dw = ctx.needs_input_grad[0], ctx.needs_input_grad[1]
        if not (need_dx or need_dw):
            return None, None, None, None, None, None
        per_row = ctx.reduction == "none"
        g = g.reshape(-1).float().contiguous()
        count = stats[1:] if ctx.reduction == "mean" else None
        C = chunk_rows(V)
        buf = torch.empty((min(C, N), V), dtype=torch.bfloat16, device=dev)
        dx = torch.empty((N, D), dtype=torch.bfloat16, device=dev) if need_dx else None
        multi = N > C
        acc = torch.empty((V, D), dtype=torch.float32, device=dev) if need_dw and multi else None
        dw = None
        st = torch.cuda.current_stream(dev).cuda_stream
        for c0 in range(0, N, C):
            rows = min(C, N - c0)
            dl = buf[:rows]
            _ck(_lib.b200dp_xent_grad(x2.data_ptr(), weight.data_ptr(), t.data_ptr(), lse.data_ptr(), g.data_ptr(),
                                      int(per_row), count.data_ptr() if count is not None else None, dl.data_ptr(),
                                      c0, rows, N, D, V, ctx.ignore_index, int(ctx.max_ctas), st),
                "b200dp_xent_grad")
            counters.bump("xent_grad")
            if need_dx:
                _gemm.gemm(dl, weight, dx[c0:c0 + rows], rows, D, V, b_mn=True)
            if need_dw:
                xc = x2[c0:c0 + rows]
                if not multi:
                    dw = _gemm.wgrad(dl, xc, V, D, rows, weight.dtype, owner=weight)
                else:
                    _gemm.gemm(dl, xc, acc, V, D, rows, a_mn=True, b_mn=True, out_mode=2 if c0 == 0 else 1,
                               splits=_gemm._splits_for(V, D, rows))
        del buf
        if need_dw and multi:
            # the chunks' fp32 sum, rounded to the weight's dtype once
            dst, accumulate, done = grad_sink.begin(weight)
            if dst is not None and dst.dtype == weight.dtype:
                if accumulate:
                    acc.add_(dst.view(V, D))
                dst.view(V, D).copy_(acc)
                done()
            else:
                dw = acc.to(weight.dtype)
        return (dx.view(ctx.x_shape) if dx is not None else None), dw, None, None, None, None


def linear_cross_entropy(x, weight, targets, ignore_index: int = -100, reduction: str = "mean",
                         max_ctas: int = 0):
    """``F.cross_entropy(F.linear(x, weight).float(), targets)`` on the fused kernels (see the module
    docstring); ``supported`` must hold.  ``max_ctas`` > 0 caps the persistent grids (tests)."""
    return _LinearXentFn.apply(x, weight, targets, ignore_index, reduction, max_ctas)
