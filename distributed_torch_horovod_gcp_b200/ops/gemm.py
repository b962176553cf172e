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
    lib.b200dp_gemm_last_error.restype = ctypes.c_char_p
    have["gemm"] = True
    have["linear"] = True


def gemm(a: torch.Tensor, b: torch.Tensor, out: torch.Tensor, M: int, N: int, K: int, *,
         a_mn: bool = False, b_mn: bool = False, bias: Optional[torch.Tensor] = None,
         residual: Optional[torch.Tensor] = None, preact: Optional[torch.Tensor] = None,
         act: int = 0, out_mode: int = 0, alpha: float = 1.0, splits: int = 1, block_n: int = 0,
         max_ctas: int = 0, stats: Optional[torch.Tensor] = None,
         res_mask: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Raw kernel call.  ``a``: [M,K] (K-major) or [K,M] (MN-major) bf16 with contiguous rows;
    ``b``: [N,K] or [K,N]; ``out``: [M,N] bf16 (out_mode 0), or bf16 / fp32 (1: add, 2: store; rounded once
    from the fp32 result).  Split-K (out_mode 1/2, splits > 1) sums in split order through an fp32 workspace
    allocated per launch on the current stream, so it may run on any stream.  ``stats`` accumulates through one per-library set of
    per-CTA slots: calls with ``stats`` (and the BatchNorm reductions of ``ops.bn``) must not run
    concurrently on different streams."""
    assert _lib is not None, "libb200dp_kernels.so not loaded"
    assert a.dtype == torch.bfloat16 and b.dtype == torch.bfloat16
    assert a.stride(-1) == 1 and b.stride(-1) == 1 and out.stride(-1) == 1
    assert out.dtype == torch.bfloat16 or (out_mode != 0 and out.dtype == torch.float32)
    bias_bf = bias.data_ptr() if bias is not None and bias.dtype == torch.bfloat16 else None
    bias_f32 = bias.data_ptr() if bias is not None and bias.dtype == torch.float32 else None
    rc = _lib.b200dp_gemm_bf16(
        a.data_ptr(), b.data_ptr(), out.data_ptr(), M, N, K, a.stride(0), b.stride(0), out.stride(0),
        int(a_mn), int(b_mn), bias_bf, bias_f32,
        residual.data_ptr() if residual is not None else None,
        preact.data_ptr() if preact is not None else None,
        act, out_mode, int(out.dtype == torch.bfloat16), float(alpha), splits, block_n, max_ctas,
        stats.data_ptr() if stats is not None else None,
        res_mask.data_ptr() if res_mask is not None else None,
        torch.cuda.current_stream(a.device).cuda_stream)
    if rc != 0:
        raise RuntimeError("b200dp_gemm_bf16: " + (_lib.b200dp_gemm_last_error() or b"").decode())
    counters.bump("gemm_sm90")
    return out


def supported(x: torch.Tensor, weight: torch.Tensor) -> bool:
    if _lib is None or x.dtype != torch.bfloat16 or weight.dtype != torch.bfloat16:
        return False
    N, K = weight.shape
    return N % 8 == 0 and K % 8 == 0 and x.shape[-1] == K and x.numel() // K >= 1


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


class _LinearFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, weight, bias, act, residual, owner=None, box=None, stats=None, park=None):
        K = weight.shape[1]
        ctx.owner = owner if owner is not None else weight
        ctx.box = box if (box is not None and ctx.needs_input_grad[0]) else None
        ctx.park = park if ctx.needs_input_grad[0] else None
        if ctx.box is not None:
            ctx.box.armed = True
        if ctx.needs_input_grad[1]:
            grad_sink.note_forward(ctx.owner)
        N = weight.shape[0]
        x2 = x.reshape(-1, K)
        if x2.stride(-1) != 1 or (x2.stride(0) % 8) or (x2.data_ptr() % 16):
            x2 = x2.contiguous()
        M = x2.shape[0]
        y = torch.empty((M, N), dtype=torch.bfloat16, device=x.device)
        need_z = act != 0 and (x.requires_grad or weight.requires_grad)
        z = torch.empty_like(y) if need_z else None
        r2 = None
        if residual is not None:
            r2 = residual.reshape(-1, N)
            if not r2.is_contiguous():
                r2 = r2.contiguous()
        gemm(x2, weight, y, M, N, K, bias=bias, residual=r2, preact=z, act=act, stats=stats)
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
        dy2 = dy.reshape(M, N)
        if not dy2.is_contiguous():
            dy2 = dy2.contiguous()
        dres = dy2.view(*ctx.x_shape[:-1], N) if ctx.has_res else None
        if ctx.act != 0:
            dz = act_backward(dy2, z, ctx.act)
        else:
            dz = dy2
        dx = dw = db = None
        if ctx.needs_input_grad[0]:
            dx = torch.empty((M, K), dtype=torch.bfloat16, device=dy.device)
            skip = skip_mask = None
            if ctx.box is not None:
                skip, skip_mask = ctx.box.take()    # skip-connection gradient of the same block input
            if skip is not None:
                if skip.dim() == 4:                 # NHWC activation -> its [M, C] matrix (a view)
                    skip = skip.permute(0, 2, 3, 1).reshape(M, K)
                else:
                    skip = skip.reshape(M, K)
                if not skip.is_contiguous():
                    skip = skip.contiguous()
                if skip_mask is not None and (K % 64):      # kernel limit: apply the sign bits here
                    bits = (skip_mask.view(M, K // 8, 1) >> torch.arange(8, device=skip.device, dtype=torch.uint8)) & 1
                    skip = skip * bits.view(M, K).to(skip.dtype)
                    skip_mask = None
            gemm(dz, weight, dx, M, K, N, b_mn=True, residual=skip, res_mask=skip_mask)   # dx = dz @ W (+ skip)
            dx = dx.view(ctx.x_shape)
            if ctx.park is not None and ctx.park.park(dx):
                dx = None                           # the block's first conv adds it in its dgrad epilogue
        if ctx.needs_input_grad[1]:
            dw = wgrad(dz, x2, N, K, M, weight.dtype, owner=ctx.owner)     # dW = dz^T @ x
        if ctx.has_bias and ctx.needs_input_grad[2]:
            db = bias_grad(dz, N, M, ctx.bias_dtype)
        return dx, dw, db, None, dres, None, None, None, None


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
        x2 = x.reshape(-1, D)
        if not x2.is_contiguous():
            x2 = x2.contiguous()
        M = x2.shape[0]
        dev = x.device
        z = torch.empty((M, Hd), dtype=torch.bfloat16, device=dev)
        h = torch.empty((M, Hd), dtype=torch.bfloat16, device=dev)
        gemm(x2, w1, h, M, Hd, D, bias=b1, preact=z, act=2)
        out = torch.empty((M, w2.shape[0]), dtype=torch.bfloat16, device=dev)
        r2 = residual.reshape(M, -1) if residual is not None else None
        if r2 is not None and not r2.is_contiguous():
            r2 = r2.contiguous()
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
        dy2 = dy.reshape(M, Do)
        if not dy2.is_contiguous():
            dy2 = dy2.contiguous()
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
        x2 = x.reshape(-1, D)
        if not x2.is_contiguous():
            x2 = x2.contiguous()
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
            g2 = g.reshape(M, Dh)
            if not g2.is_contiguous() or g2.data_ptr() % 16:
                g2 = g2.contiguous()
            gs.append(g2)
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


def linear(x, weight, bias=None, act: Optional[str] = None, residual=None, owner=None, box=None, stats=None,
           park=None):
    """``owner``: the parameter whose storage ``weight`` is a 2D view of (a 1x1 conv weight), so the
    weight gradient can be written into its gradient-bucket slot directly.  ``box``: a
    ``grad_sink.GradBox`` through which a later node hands this layer the skip-connection gradient of
    the same input (added in the dgrad epilogue)."""
    return _LinearFn.apply(x, weight, bias, ACT[act], residual, owner, box, stats, park)
