"""wgmma GEMM binding (csrc/gemm_sm90.cu) and the autograd ``linear`` built on it.

    y = act(x @ W^T + b) (+ residual)          forward : A = x (K-major),  B = W (K-major)
    dx = dy' @ W                                dgrad   : A = dy' (K-major), B = W (MN-major)
    dW = dy'^T @ x                              wgrad   : A = dy' (MN-major), B = x (MN-major),
                                                          split-K, partials summed in split order
No transposes are materialised: the kernel takes MN-major operands through its GMMA
descriptors.  ``dy' = dy * act'(z)`` is fused into the dgrad of the *next* layer's epilogue
where possible; here it is computed by the epilogue modes 3/4 of the kernel when the layer
has an activation.
"""
from __future__ import annotations

import ctypes
from typing import Optional

import torch

from . import counters
from . import grad_sink

_lib = None
ACT = {None: 0, "none": 0, "relu": 1, "gelu": 2}


def register(lib, have):
    global _lib
    if not hasattr(lib, "b200dp_gemm_bf16"):
        return
    _lib = lib
    vp, i, f = ctypes.c_void_p, ctypes.c_int, ctypes.c_float
    lib.b200dp_gemm_bf16.argtypes = [vp, vp, vp, i, i, i, i, i, i, i, i, vp, vp, vp, vp, i, i, i, f, i,
                                     i, i, vp, vp, ctypes.c_uint64]
    lib.b200dp_gemm_bf16.restype = i
    if hasattr(lib, "b200dp_gemm_bf16_scaled"):
        lib.b200dp_gemm_bf16_scaled.argtypes = [vp, vp, vp, i, i, i, i, i, i, i, i, vp, vp, vp, vp, i, i, i, f, f,
                                                i, i, i, vp, vp, ctypes.c_uint64]
        lib.b200dp_gemm_bf16_scaled.restype = i
        have["gemm_scaled"] = True
    lib.b200dp_gemm_last_error.restype = ctypes.c_char_p
    have["gemm"] = True
    have["linear"] = True


def gemm(a: torch.Tensor, b: torch.Tensor, out: torch.Tensor, M: int, N: int, K: int, *,
         a_mn: bool = False, b_mn: bool = False, bias: Optional[torch.Tensor] = None,
         residual: Optional[torch.Tensor] = None, preact: Optional[torch.Tensor] = None,
         act: int = 0, out_mode: int = 0, alpha: float = 1.0, splits: int = 1, block_n: int = 0,
         max_ctas: int = 0, stats: Optional[torch.Tensor] = None,
         res_mask: Optional[torch.Tensor] = None, beta: float = 1.0) -> torch.Tensor:
    """Raw kernel call.  ``a``: [M,K] (K-major) or [K,M] (MN-major) bf16 with contiguous rows;
    ``b``: [N,K] or [K,N]; ``out``: [M,N] bf16 (out_mode 0), or bf16 / fp32 (1: add, 2: store; rounded once
    from the fp32 result).  Split-K (out_mode 1/2, splits > 1) sums in split order through an fp32 workspace
    allocated per launch on the current stream, so it may run on any stream.  ``stats`` accumulates through one per-library set of
    per-CTA slots: calls with ``stats`` (and the BatchNorm reductions of ``ops.bn``) must not run
    concurrently on different streams.  ``beta`` multiplies the residual (``act(alpha AB + bias) + beta residual``,
    rounded once); ``beta != 1`` needs a plain residual (act 0..2, no ``res_mask``)."""
    assert _lib is not None, "libb200dp_kernels.so not loaded"
    assert a.dtype == torch.bfloat16 and b.dtype == torch.bfloat16
    assert a.stride(-1) == 1 and b.stride(-1) == 1 and out.stride(-1) == 1
    assert out.dtype == torch.bfloat16 or (out_mode != 0 and out.dtype == torch.float32)
    bias_bf = bias.data_ptr() if bias is not None and bias.dtype == torch.bfloat16 else None
    bias_f32 = bias.data_ptr() if bias is not None and bias.dtype == torch.float32 else None
    head = (a.data_ptr(), b.data_ptr(), out.data_ptr(), M, N, K, a.stride(0), b.stride(0), out.stride(0),
            int(a_mn), int(b_mn), bias_bf, bias_f32,
            residual.data_ptr() if residual is not None else None,
            preact.data_ptr() if preact is not None else None,
            act, out_mode, int(out.dtype == torch.bfloat16), float(alpha))
    tail = (splits, block_n, max_ctas,
            stats.data_ptr() if stats is not None else None,
            res_mask.data_ptr() if res_mask is not None else None,
            torch.cuda.current_stream(a.device).cuda_stream)
    if beta == 1.0:
        rc = _lib.b200dp_gemm_bf16(*head, *tail)
    else:
        rc = _lib.b200dp_gemm_bf16_scaled(*head, float(beta), *tail)
    if rc != 0:
        raise RuntimeError("b200dp_gemm_bf16: " + (_lib.b200dp_gemm_last_error() or b"").decode())
    counters.bump("gemm_sm90")
    return out


def _weight_ok(w: torch.Tensor, dev) -> bool:
    """A bf16 [N, K] operand the TMA descriptor takes as it is: unit column stride, 16-byte rows and base."""
    return (w.dtype == torch.bfloat16 and w.dim() == 2 and w.device == dev and w.shape[0] % 8 == 0
            and w.shape[1] % 8 == 0 and w.stride(1) == 1 and w.stride(0) % 8 == 0 and w.data_ptr() % 16 == 0)


def _bias_ok(bias: Optional[torch.Tensor], N: int, dev) -> bool:
    """The epilogue reads ``bias[col]`` for col < N in bf16 or fp32 (any other dtype would not be passed)."""
    return bias is None or (bias.dtype in (torch.bfloat16, torch.float32) and bias.device == dev
                            and tuple(bias.shape) == (N,) and bias.stride(0) == 1)


def _residual_ok(residual: Optional[torch.Tensor], shape, dev) -> bool:
    """The epilogue reads the residual as a bf16 [M, N] matrix, so it must be one of the output's shape (no
    broadcasting).  A misaligned or strided one is copied into a dense tensor first (``_dense``)."""
    return residual is None or (residual.dtype == torch.bfloat16 and residual.device == dev
                                and tuple(residual.shape) == tuple(shape))


def supported(x: torch.Tensor, weight: torch.Tensor, bias: Optional[torch.Tensor] = None,
              residual: Optional[torch.Tensor] = None, w2: Optional[torch.Tensor] = None,
              b2: Optional[torch.Tensor] = None) -> bool:
    """Whether ``linear(x, weight, bias, residual=residual)`` (or ``qkv_proj``) runs on the kernel: bf16 ``x``
    with at least one row and bf16 weights of whole 16-byte rows, a bias of N elements in bf16 or fp32, and a bf16
    residual of the output's shape.  With ``w2`` (``mlp``): fc1 = (weight, bias) and fc2 = (w2, b2), and the
    residual is added to fc2's output."""
    if _lib is None or x.dtype != torch.bfloat16 or x.dim() < 1 or not _weight_ok(weight, x.device):
        return False
    N, K = weight.shape
    if x.shape[-1] != K or x.numel() // K < 1 or not _bias_ok(bias, N, x.device):
        return False
    if w2 is not None:
        if not (_weight_ok(w2, x.device) and w2.shape[1] == N and _bias_ok(b2, w2.shape[0], x.device)):
            return False
        N = w2.shape[0]
    return _residual_ok(residual, (*x.shape[:-1], N), x.device)


def _dense(t: torch.Tensor) -> torch.Tensor:
    """``t`` as a contiguous matrix with a 16-byte aligned base (``contiguous`` keeps a contiguous view at an
    unaligned storage offset as it is)."""
    if t.is_contiguous() and t.data_ptr() % 16 == 0:
        return t
    return t.clone(memory_format=torch.contiguous_format)


def _splits_for(M_out: int, N_out: int, K_red: int, sms: int = 132) -> int:
    tiles = ((M_out + 127) // 128) * ((N_out + 127) // 128)
    if tiles >= (2 * sms) // 3:
        return 1                       # enough tiles to fill the GPU: no split, direct bf16 store
    kb = (K_red + 63) // 64
    want = max(1, (2 * sms) // max(tiles, 1))
    return max(1, min(want, kb // 4 if kb >= 8 else 1))


_ones_cache = {}


def _ones(M: int, device) -> torch.Tensor:
    key = (M, str(device))
    t = _ones_cache.get(key)
    if t is None:
        t = torch.ones((M, 8), dtype=torch.bfloat16, device=device)
        _ones_cache[key] = t
    return t


def wgrad(dz: torch.Tensor, x2: torch.Tensor, N: int, K: int, M: int, dtype, owner=None):
    """dW[N,K] = dz[M,N]^T @ x2[M,K] with both operands MN-major (no transposes), written in ``dtype`` by the
    GEMM itself.  With ``owner`` (the parameter) carrying a grad sink the result goes straight into its
    gradient-bucket slot and ``None`` is returned (ops/grad_sink.py)."""
    dst, acc, done = grad_sink.begin(owner) if owner is not None else (None, False, None)
    if dst is not None and dst.dtype != dtype:
        dst, acc, done = None, False, None
    dw = dst.as_strided((N, K), (K, 1)) if dst is not None else torch.empty((N, K), dtype=dtype, device=dz.device)
    splits = _splits_for(N, K, M)
    if splits == 1 and dtype == torch.bfloat16:
        gemm(dz, x2, dw, N, K, M, a_mn=True, b_mn=True, residual=dw if acc else None)
    else:
        gemm(dz, x2, dw, N, K, M, a_mn=True, b_mn=True, out_mode=1 if acc else 2, splits=splits)
    if done is not None:
        done()
        return None
    return dw


def bias_grad(dz: torch.Tensor, N: int, M: int, dtype) -> torch.Tensor:
    """db[N] = column sums of dz — as a GEMM against a ones matrix (reads dz once, in bf16)."""
    acc = torch.zeros((N, 8), dtype=torch.float32, device=dz.device)
    kb = (M + 63) // 64
    gemm(dz, _ones(M, dz.device), acc, N, 8, M, a_mn=True, b_mn=True, out_mode=1,
         splits=max(1, min(kb // 4, (2 * 132) // max((N + 127) // 128, 1))), block_n=64)
    return acc[:, 0].to(dtype)


def dgrad(dz: torch.Tensor, weight: torch.Tensor, residual: Optional[torch.Tensor] = None,
          res_mask: Optional[torch.Tensor] = None) -> torch.Tensor:
    """dx[M,K] = dz[M,N] @ W[N,K] (+ ``residual`` [M,K], kept only where the bits of ``res_mask`` are set:
    ReLU sign bits, 1 byte per 8 columns)."""
    M, (N, K) = dz.shape[0], weight.shape
    if res_mask is not None and (K % 64):      # kernel limit: apply the sign bits here
        bits = (res_mask.view(M, K // 8, 1) >> torch.arange(8, device=dz.device, dtype=torch.uint8)) & 1
        residual = residual * bits.view(M, K).to(residual.dtype)
        res_mask = None
    dx = torch.empty((M, K), dtype=torch.bfloat16, device=dz.device)
    return gemm(dz, weight, dx, M, K, N, b_mn=True, residual=residual, res_mask=res_mask)


class _LinearFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, weight, bias, act, residual):
        K = weight.shape[1]
        if ctx.needs_input_grad[1]:
            grad_sink.note_forward(weight)
        N = weight.shape[0]
        x2 = x.reshape(-1, K)
        if x2.stride(-1) != 1 or (x2.stride(0) % 8) or (x2.data_ptr() % 16):
            x2 = x2.clone(memory_format=torch.contiguous_format)
        M = x2.shape[0]
        y = torch.empty((M, N), dtype=torch.bfloat16, device=x.device)
        need_z = act != 0 and any(ctx.needs_input_grad[0:3])      # dz feeds dx, dW and db; not dres
        z = torch.empty_like(y) if need_z else None
        r2 = None
        if residual is not None:
            r2 = _dense(residual.reshape(-1, N))
        gemm(x2, weight, y, M, N, K, bias=bias, residual=r2, preact=z, act=act)
        ctx.save_for_backward(x2, weight, z)
        ctx.act, ctx.has_bias, ctx.has_res = act, bias is not None, residual is not None
        ctx.x_shape = x.shape
        ctx.bias_dtype = bias.dtype if bias is not None else None
        return y.view(*x.shape[:-1], N)

    @staticmethod
    def backward(ctx, dy):
        x2, weight, z = ctx.saved_tensors
        N, K = weight.shape
        M = x2.shape[0]
        dy2 = _dense(dy.reshape(M, N))
        dres = dy2.view(*ctx.x_shape[:-1], N) if ctx.has_res else None
        if ctx.act != 0 and any(ctx.needs_input_grad[0:3]):
            dz = act_backward(dy2, z, ctx.act)
        else:
            dz = dy2
        dx = dw = db = None
        if ctx.needs_input_grad[0]:
            dx = dgrad(dz, weight).view(ctx.x_shape)                       # dx = dz @ W
        if ctx.needs_input_grad[1]:
            dw = wgrad(dz, x2, N, K, M, weight.dtype, owner=weight)        # dW = dz^T @ x
        if ctx.has_bias and ctx.needs_input_grad[2]:
            db = bias_grad(dz, N, M, ctx.bias_dtype)
        return dx, dw, db, None, dres


def act_backward(dy2: torch.Tensor, z: torch.Tensor, act: int) -> torch.Tensor:
    """dz = dy * act'(z) (stand-alone form; the MLP block fuses this into the fc2 dgrad epilogue)."""
    if act == 1:
        return dy2 * (z > 0).to(dy2.dtype)
    zf = z.float()
    cdf = 0.5 * (1.0 + torch.erf(zf * 0.7071067811865476))
    pdf = 0.3989422804014327 * torch.exp(-0.5 * zf * zf)
    return (dy2.float() * (cdf + zf * pdf)).to(torch.bfloat16)


class _MLPFn(torch.autograd.Function):
    """Transformer MLP block  out = fc2(gelu(fc1(x))) + residual  as ONE autograd node so the
    backward can fuse  dz = (dy @ W2) * gelu'(z)  into the fc2-dgrad GEMM epilogue (act mode 3)."""

    @staticmethod
    def forward(ctx, x, w1, b1, w2, b2, residual):
        D, Hd = w1.shape[1], w1.shape[0]
        x2 = _dense(x.reshape(-1, D))
        M = x2.shape[0]
        dev = x.device
        z = torch.empty((M, Hd), dtype=torch.bfloat16, device=dev)
        h = torch.empty((M, Hd), dtype=torch.bfloat16, device=dev)
        gemm(x2, w1, h, M, Hd, D, bias=b1, preact=z, act=2)
        out = torch.empty((M, w2.shape[0]), dtype=torch.bfloat16, device=dev)
        r2 = _dense(residual.reshape(M, -1)) if residual is not None else None
        gemm(h, w2, out, M, w2.shape[0], Hd, bias=b2, residual=r2)
        ctx.save_for_backward(x2, w1, w2, z, h)
        ctx.owners = (w1, w2)
        if ctx.needs_input_grad[1]:
            grad_sink.note_forward(w1)
        if ctx.needs_input_grad[3]:
            grad_sink.note_forward(w2)
        ctx.x_shape, ctx.has_res = x.shape, residual is not None
        ctx.bdt = (b1.dtype, b2.dtype)
        return out.view(*x.shape[:-1], w2.shape[0])

    @staticmethod
    def backward(ctx, dy):
        x2, w1, w2, z, h = ctx.saved_tensors
        M, D = x2.shape
        Hd, Do = w1.shape[0], w2.shape[0]
        dy2 = _dense(dy.reshape(M, Do))
        dev = dy.device
        dz = torch.empty((M, Hd), dtype=torch.bfloat16, device=dev)
        gemm(dy2, w2, dz, M, Hd, Do, b_mn=True, residual=z, act=3)        # (dy @ W2) * gelu'(z)
        dw2 = wgrad(dy2, h, Do, Hd, M, w2.dtype, owner=ctx.owners[1])
        db2 = bias_grad(dy2, Do, M, ctx.bdt[1])
        dw1 = wgrad(dz, x2, Hd, D, M, w1.dtype, owner=ctx.owners[0])
        db1 = bias_grad(dz, Hd, M, ctx.bdt[0])
        dx = torch.empty((M, D), dtype=torch.bfloat16, device=dev)
        gemm(dz, w1, dx, M, D, Hd, b_mn=True)
        dres = dy2.view(*ctx.x_shape[:-1], Do) if ctx.has_res else None
        return dx.view(ctx.x_shape), dw1, db1, dw2, db2, dres


def mlp(x, w1, b1, w2, b2, residual=None):
    return _MLPFn.apply(x, w1, b1, w2, b2, residual)


class _QKVFn(torch.autograd.Function):
    """Attention input projection producing q, k, v as three DENSE [M, D] matrices (three GEMMs on
    row-slices of the packed [3D, D] weight).  A packed [M, 3D] output forces PyTorch to un-pack
    with strided views forward and to re-pack dq/dk/dv with a cat + copies backward.  Here the
    backward consumes
    dq, dk, dv where they are: dx is accumulated through the GEMM's residual input and the weight
    gradient is written slice by slice."""

    @staticmethod
    def forward(ctx, x, weight, bias):
        D3, D = weight.shape
        Dh = D3 // 3
        x2 = _dense(x.reshape(-1, D))
        M = x2.shape[0]
        outs = []
        for i in range(3):
            o = torch.empty((M, Dh), dtype=torch.bfloat16, device=x.device)
            gemm(x2, weight[i * Dh:(i + 1) * Dh], o, M, Dh, D,
                 bias=bias[i * Dh:(i + 1) * Dh] if bias is not None else None)
            outs.append(o.view(*x.shape[:-1], Dh))
        ctx.save_for_backward(x2, weight)
        ctx.x_shape, ctx.has_bias = x.shape, bias is not None
        ctx.bdt = bias.dtype if bias is not None else None
        return tuple(outs)

    @staticmethod
    def backward(ctx, dq, dk, dv):
        x2, weight = ctx.saved_tensors
        D3, D = weight.shape
        Dh = D3 // 3
        M = x2.shape[0]
        dev = x2.device
        gs = []
        for g in (dq, dk, dv):
            gs.append(_dense(g.reshape(M, Dh)))
        dx = None
        if ctx.needs_input_grad[0]:
            for i, g2 in enumerate(gs):
                nxt = torch.empty((M, D), dtype=torch.bfloat16, device=dev)
                gemm(g2, weight[i * Dh:(i + 1) * Dh], nxt, M, D, Dh, b_mn=True, residual=dx)
                dx = nxt
            dx = dx.view(ctx.x_shape)
        dw = db = None
        if ctx.needs_input_grad[1]:
            dw = torch.empty((D3, D), dtype=weight.dtype, device=dev)
            for i, g2 in enumerate(gs):
                dw[i * Dh:(i + 1) * Dh].copy_(wgrad(g2, x2, Dh, D, M, weight.dtype))
        if ctx.has_bias and ctx.needs_input_grad[2]:
            db = torch.cat([bias_grad(g2, Dh, M, ctx.bdt) for g2 in gs])
        return dx, dw, db


def qkv_proj(x, weight, bias):
    return _QKVFn.apply(x, weight, bias)


def linear(x, weight, bias=None, act: Optional[str] = None, residual=None):
    return _LinearFn.apply(x, weight, bias, ACT[act], residual)
