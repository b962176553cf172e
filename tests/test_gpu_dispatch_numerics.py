"""Each public op of ``ops.functional`` on both sides of its dispatch predicate, under the launch guard
(``launch_guard.py``): every kernel launch is checked on the host first, so an input a predicate wrongly accepts
shows up as a ``GuardError`` (a pointer past its allocation, a misaligned vector load) and never reaches the GPU.

Every case states the path it must take and checks three things:
1. the path: the guard's per-symbol launch counts (kernel path: the launches it expects; reference path: none);
2. kernel path: the output and every gradient against float64 of what the op means on the exact stored inputs,
   with the existing bounds (``epilogue_bounds`` and the per-launch checks of ``test_gpu_autograd_numerics``,
   ``ln_bounds``, ``attn_fwd_bounds``, ``xent_fwd_bounds``, the BatchNorm bounds);
3. reference path: bit for bit what the ``*_reference`` composition (or the torch module) gives on the same
   inputs, gradients and module state included; where the reference raises, the op raises the same type.

The CPU self-tests at the end feed the guard's checker fake allocations and arguments, one per violation class."""
import copy
import math
from types import SimpleNamespace

import pytest
import torch
import torch.nn.functional as F
from torch import nn

import launch_guard
from fp64_bounds import U32, assert_within_bound, report_ratios
from launch_guard import GuardError
from test_gpu_autograd_numerics import Spy, check_launches
from test_gpu_resnet_numerics import (FLUSH, _pad64, bf16_store, bn_stat_bounds, epilogue_bounds,
                                      running_stats_bounds)
from test_gpu_vit_numerics import attn_fwd_bounds, ln_bounds
from test_gpu_lm_loss import xent_fwd_bounds

gpu = pytest.mark.gpu
BF16, F16, F32 = torch.bfloat16, torch.float16, torch.float32
GEMM, BN_FWD, BN_BWD, BN_APPLY = "b200dp_gemm_bf16", "b200dp_bn_fwd", "b200dp_bn_bwd", "b200dp_bn_apply"
LN_FWD, LN_BWD = "b200dp_ln_fwd", "b200dp_ln_bwd"


@pytest.fixture(scope="module", autouse=True)
def _report_ratios():
    yield
    report_ratios()


@pytest.fixture
def env(monkeypatch):
    from distributed_torch_horovod_gcp_b200.ops import bn, bottleneck, conv, functional, gemm, grad_sink, kernels
    assert kernels.has("gemm") and kernels.has("conv_bn_act") and kernels.has("layer_norm"), \
        "libb200dp_kernels.so not loaded"
    monkeypatch.setattr(functional, "_FORCE_REFERENCE", False)
    calls = launch_guard.install(monkeypatch)
    ops = SimpleNamespace(gemm=gemm, conv=conv, bn=bn, bottleneck=bottleneck, grad_sink=grad_sink)
    return SimpleNamespace(F2=functional, calls=calls, spy=Spy(monkeypatch, ops), ops=ops)


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _randn(shape, seed, dtype=BF16, scale=1.0):
    """Seeded CPU normal values, rounded to ``dtype``, moved to the GPU."""
    return (scale * torch.randn(shape, generator=_gen(seed))).to(dtype).cuda()


def _at_offset(t, elems):
    """A copy of ``t`` stored ``elems`` elements into a larger buffer: a view at that storage offset."""
    buf = torch.zeros(t.numel() + elems + 8, dtype=t.dtype, device=t.device)
    v = buf[elems:elems + t.numel()].view(t.shape)
    v.copy_(t)
    return v


def _fwd_bwd(fn, make, seed):
    """``fn(*args)`` for ``args, leaves = make()``, then the backward of a seeded gradient of the output's dtype.
    Returns the output and the gradients of the leaves (in order)."""
    args, leaves = make()
    out = fn(*args)
    if out.requires_grad:
        dy = torch.randn(out.shape, generator=_gen(seed)).to(out.dtype).cuda()
        out.backward(dy)
    torch.cuda.synchronize()
    return out.detach(), [l.grad for l in leaves], args


def _same(a, b, what):
    assert (a is None) == (b is None), f"{what}: one side is None"
    if a is not None:
        assert a.dtype == b.dtype and a.shape == b.shape, f"{what}: {a.dtype} {tuple(a.shape)} vs {b.dtype} " \
                                                          f"{tuple(b.shape)}"
        assert torch.equal(a, b) or bool(((a == b) | (a.isnan() & b.isnan())).all()), f"{what} differs"


def _expect_reference(env, op, ref, make, seed=1):
    """The op takes the reference path: no launch reached the guard, and output and gradients are ``ref``'s bits."""
    torch.manual_seed(0)
    out, grads, _ = _fwd_bwd(op, make, seed)
    assert sum(env.calls.values()) == 0, f"reference path expected, the guard saw {dict(env.calls)}"
    torch.manual_seed(0)
    rout, rgrads, _ = _fwd_bwd(ref, make, seed)
    _same(out, rout, "output")
    for i, (g, rg) in enumerate(zip(grads, rgrads)):
        _same(g, rg, f"grad {i}")


def _expect_raise(env, op, ref, make):
    args, _ = make()
    with pytest.raises(Exception) as want:
        ref(*args)
    with pytest.raises(want.type):
        op(*make()[0])
    assert sum(env.calls.values()) == 0, f"the guard saw {dict(env.calls)} before the error"


def _expect_kernel(env, symbols):
    for s in symbols:
        assert env.calls[s] > 0, f"kernel path expected: no {s} launch went through the guard ({dict(env.calls)})"


# ================================================================================================ linear
def _linear_make(M, N, K, x="plain", bdt=BF16, res=None, wform="plain", xdt=BF16, blen=None, seed=0):
    """x [M, K] (``x`` form: plain, 3d, strided rows, storage offset 8 or 1 elements), w [N, K] (or the transpose
    of a [K, N] tensor), bias of ``bdt`` with ``blen`` elements, residual (None, bf16, fp32, bcastN, bcast1N,
    offset1: a bf16 one at a 2-byte storage offset)."""
    def make():
        xv = _randn((M, K + 8), seed, xdt)
        xl = xv[:, :K].contiguous() if x != "strided" else xv
        xl.requires_grad_(True)
        wl = _randn((K, N) if wform == "transposed" else (N, K), seed + 1, BF16 if wform != "fp32" else F32,
                    1 / math.sqrt(K)).requires_grad_(True)
        bl = _randn((blen or N,), seed + 2, bdt).requires_grad_(True) if bdt is not None else None
        rl = None
        if res is not None:
            shape = {"bcastN": (N,), "bcast1N": (1, N)}.get(res, (M, N))
            rl = _randn(shape, seed + 3, F32 if res == "fp32" else BF16).requires_grad_(True)
        xa = {"strided": lambda: xl[:, :K], "3d": lambda: xl.view(1, M, K),
              "off8": lambda: _at_offset(xl, 8), "off1": lambda: _at_offset(xl, 1)}.get(x, lambda: xl)()
        wa = wl.t() if wform == "transposed" else wl
        ra = _at_offset(rl, 1) if res == "offset1" else rl
        if ra is not None and x == "3d":
            ra = ra.view(1, M, N) if ra.dim() == 2 and ra.shape[0] == M else ra
        args = (xa, wa, bl, None, ra)
        return args, [t for t in (xl, wl, bl, rl) if t is not None]
    return make


def _linear_e2e(x2, w, b, r2, dy2, out2, grads, need_b, need_r):
    """Kernel path, no activation: y, dx, dW, db against float64 of the node on its exact inputs."""
    (y, E), _ = epilogue_bounds(x2, w, 1.0, b, 0, r2)
    assert_within_bound(out2, y, group="linear e2e y", terms=[(1.0, E)])
    gx, gw = grads[0][..., :x2.shape[1]].reshape(x2.shape), grads[1]
    (dx, Edx), _ = epilogue_bounds(dy2, w.t())
    assert_within_bound(gx, dx, group="linear e2e dx", terms=[(1.0, Edx)])
    (dw, Edw), _ = epilogue_bounds(dy2.t(), x2.t())
    assert_within_bound(gw, dw, group="linear e2e dW", terms=[(1.0, Edw)])
    i = 2
    if need_b:
        ref = dy2.double().sum(0)
        Eb = 2 * _pad64(x2.shape[0]) * U32 * dy2.double().abs().sum(0) + FLUSH
        assert_within_bound(grads[i], ref, group="linear e2e db",
                            terms=[(1.0, bf16_store(Eb, ref) if b.dtype == BF16 else Eb)])
        i += 1
    if need_r:
        _same(grads[i].reshape(dy2.shape), dy2, "residual gradient is dy")


# id, make kwargs, expected path, M, N, K
LINEAR_KERNEL = [
    ("bf16-bias", dict(), 64, 72, 40),
    ("fp32-bias", dict(bdt=F32), 64, 72, 40),
    ("no-bias-M1", dict(bdt=None), 1, 8, 8),
    ("bf16-residual", dict(res="bf16"), 33, 16, 24),
    ("residual-offset-2B", dict(res="offset1"), 33, 16, 24),
    ("x-3d", dict(x="3d", bdt=F32, res="bf16"), 7, 24, 16),
    ("x-strided-rows", dict(x="strided"), 20, 16, 32),
    ("x-offset-16B", dict(x="off8"), 20, 16, 32),
    ("x-offset-2B", dict(x="off1"), 20, 16, 32),
]


@gpu
@pytest.mark.parametrize("cid,kw,M,N,K", LINEAR_KERNEL, ids=[c[0] for c in LINEAR_KERNEL])
def test_linear_kernel_path(cid, kw, M, N, K, env):
    make = _linear_make(M, N, K, seed=M + N, **kw)
    out, grads, args = _fwd_bwd(env.F2.linear, make, seed=3)
    _expect_kernel(env, [GEMM])
    check_launches(env.spy, f"linear {cid}")
    x, w, b, _, r = args
    x2 = x.detach().reshape(-1, K)
    dy2 = torch.randn(out.shape, generator=_gen(3)).to(BF16).cuda().reshape(-1, N)
    r2 = r.detach().reshape(-1, N) if r is not None else None
    _linear_e2e(x2, w.detach(), b.detach() if b is not None else None, r2, dy2, out.reshape(-1, N), grads,
                b is not None, r is not None)


LINEAR_REFERENCE = [
    ("fp16-bias", dict(bdt=F16), 16, 24, 16),
    ("fp32-residual", dict(res="fp32"), 16, 24, 16),
    ("bcast-residual-N", dict(res="bcastN"), 16, 24, 16),
    ("bcast-residual-1xN", dict(res="bcast1N"), 16, 24, 16),
    ("x-fp16", dict(xdt=F16, bdt=F16), 16, 24, 16),
    ("x-fp32", dict(xdt=F32, bdt=F32), 16, 24, 16),
    ("N-not-mult-8", dict(), 16, 20, 16),
    ("K-not-mult-8", dict(), 16, 24, 12),
    ("weight-transposed", dict(wform="transposed"), 16, 24, 16),
    ("weight-fp32-bias-bf16", dict(wform="fp32"), 16, 24, 16),
    ("empty-batch", dict(), 0, 24, 16),
]


@gpu
@pytest.mark.parametrize("cid,kw,M,N,K", LINEAR_REFERENCE, ids=[c[0] for c in LINEAR_REFERENCE])
def test_linear_reference_path(cid, kw, M, N, K, env):
    _expect_reference(env, env.F2.linear, env.F2.linear_reference, _linear_make(M, N, K, seed=M + N, **kw))


@gpu
def test_linear_wrong_length_bias_raises(env):
    _expect_raise(env, env.F2.linear, env.F2.linear_reference, _linear_make(16, 24, 16, blen=16))


# ================================================================================================ MLP
def _mlp_make(M, D, Hd, Do, b1dt=BF16, b2dt=BF16, w2dt=BF16, res=False, seed=0):
    def make():
        x = _randn((M, D), seed).requires_grad_(True)
        w1 = _randn((Hd, D), seed + 1, BF16, 1 / math.sqrt(D)).requires_grad_(True)
        b1 = _randn((Hd,), seed + 2, b1dt).requires_grad_(True)
        w2 = _randn((Do, Hd), seed + 3, w2dt, 1 / math.sqrt(Hd)).requires_grad_(True)
        b2 = _randn((Do,), seed + 4, b2dt).requires_grad_(True)
        r = _randn((M, Do), seed + 5).requires_grad_(True) if res else None
        return (x, w1, b1, w2, b2, r), [t for t in (x, w1, b1, w2, b2, r) if t is not None]
    return make


def _mlp_ref(x, w1, b1, w2, b2, r):
    from distributed_torch_horovod_gcp_b200.ops import functional as F2
    return F2.linear_reference(F2.linear_reference(x, w1, b1, act="gelu"), w2, b2, residual=r)


MLP_CASES = [   # id, kwargs, kernel?
    ("bf16", dict(res=True), True),
    ("fp32-biases-M1", dict(M=1, b1dt=F32, b2dt=F32), True),
    ("fp16-b1", dict(b1dt=F16), False),
    ("fp16-b2", dict(b2dt=F16), False),
    ("fp32-w2", dict(w2dt=F32), False),
    ("Do-not-mult-8", dict(Do=20), False),
]


@gpu
@pytest.mark.parametrize("cid,kw,kernel", MLP_CASES, ids=[c[0] for c in MLP_CASES])
def test_mlp_dispatch(cid, kw, kernel, env):
    shape, kw = dict(M=9, D=32, Hd=64, Do=32), dict(kw)
    shape.update({k: kw.pop(k) for k in list(kw) if k in shape})
    make = _mlp_make(**shape, **kw, seed=11)
    if not kernel:
        _expect_reference(env, env.F2.mlp, _mlp_ref, make)
        return
    out, grads, args = _fwd_bwd(env.F2.mlp, make, seed=4)
    _expect_kernel(env, [GEMM])
    check_launches(env.spy, f"mlp {cid}")
    # the node's output is fc2's launch output, and it had both biases
    fwd = [r for r in env.spy.of("gemm") if not r.a_mn and not r.b_mn]
    assert len(fwd) == 2 and fwd[0].bias is args[2] and fwd[1].bias is args[4]
    _same(out.reshape(fwd[1].out.shape), fwd[1].out, "mlp output is fc2's")


# ================================================================================================ QKV + attention
def _qkv_make(B, S, D, bdt=BF16, seed=0):
    def make():
        x = _randn((B, S, D), seed).requires_grad_(True)
        w = _randn((3 * D, D), seed + 1, BF16, 1 / math.sqrt(D)).requires_grad_(True)
        b = _randn((3 * D,), seed + 2, bdt).requires_grad_(True) if bdt is not None else None
        return (x, w, b), [t for t in (x, w, b) if t is not None]
    return make


@gpu
@pytest.mark.parametrize("bdt", [BF16, F32], ids=["bf16-bias", "fp32-bias"])
def test_qkv_attention_kernel_path(bdt, env):
    """hd = 64: the three projections on the GEMM, then the flash-attention kernels."""
    B, S, D, H = 2, 65, 128, 2
    make = _qkv_make(B, S, D, bdt, seed=21)
    out, grads, (x, w, b) = _fwd_bwd(lambda x, w, b: env.F2.qkv_attention(x, w, b, H), make, seed=5)
    _expect_kernel(env, [GEMM, "b200dp_attn_fwd_ex", "b200dp_attn_bwd"])
    check_launches(env.spy, "qkv")
    fwd = [r for r in env.spy.of("gemm") if not r.a_mn and not r.b_mn][:3]
    qkv = [r.out.view(B, S, H, 64).transpose(1, 2) for r in fwd]
    for i, r in enumerate(fwd):
        assert r.bias is not None and r.bias.data_ptr() == b.data_ptr() + i * D * b.element_size()
    o64, _, o_terms, _, _ = attn_fwd_bounds(*qkv)
    assert_within_bound(out.view(B, S, H, 64).transpose(1, 2), o64, group="qkv attention o", terms=o_terms)
    assert all(g is not None and torch.isfinite(g.float()).all() for g in grads)


@gpu
def test_qkv_attention_head_dim_32_uses_sdpa(env):
    """hd = 32: the projections on the GEMM, attention in SDPA; the output is SDPA's on the GEMM's q, k, v."""
    B, S, D, H = 2, 17, 64, 2
    out, _, _ = _fwd_bwd(lambda x, w, b: env.F2.qkv_attention(x, w, b, H), _qkv_make(B, S, D, seed=22), seed=6)
    _expect_kernel(env, [GEMM])
    assert env.calls["b200dp_attn_fwd_ex"] == 0
    q, k, v = [r.out.view(B, S, H, 32).transpose(1, 2) for r in env.spy.of("gemm")[:3]]
    _same(out, F.scaled_dot_product_attention(q, k, v).transpose(1, 2).reshape(B, S, D), "SDPA on the GEMM's q, k, v")


@gpu
@pytest.mark.parametrize("bdt", [F16, None], ids=["fp16-bias", "no-bias-fp32-x"])
def test_qkv_attention_reference_path(bdt, env):
    B, S, D, H = 2, 17, 128, 2
    base = _qkv_make(B, S, D, bdt, seed=23)
    make = base
    if bdt is None:
        def make():
            (x, w, b), leaves = base()
            xf = x.detach().float().requires_grad_(True)
            return (xf, w, b), [xf, w]
    ref = lambda x, w, b: env.F2.attention_reference(env.F2.linear_reference(x, w, b), H)   # noqa: E731
    _expect_reference(env, lambda x, w, b: env.F2.qkv_attention(x, w, b, H), ref, make)


@gpu
@pytest.mark.parametrize("hd", [64, 32])
def test_packed_attention_is_the_reference(hd, env):
    """``F2.attention`` on a packed [B, S, 3D] tensor is always the SDPA composition."""
    B, S, H = 2, 33, 2

    def make():
        qkv = _randn((B, S, 3 * H * hd), 31).requires_grad_(True)
        return (qkv,), [qkv]
    _expect_reference(env, lambda t: env.F2.attention(t, H), lambda t: env.F2.attention_reference(t, H), make)


# ================================================================================================ LayerNorm
LN_EPS = 1e-6


def _ln_make(R, C, pdt=BF16, bdt=None, x="plain", weight=True, bias=True, wlen=None, xdt=BF16, seed=0):
    def make():
        g = _gen(seed)
        xl = (2 * torch.randn(R, C, generator=g) + 0.5).to(xdt).cuda().requires_grad_(True)
        w = (torch.rand(wlen or C, generator=g) + 0.5).to(pdt).cuda().requires_grad_(True) if weight else None
        b = (0.1 * torch.randn(C, generator=g)).to(bdt or pdt).cuda().requires_grad_(True) if bias else None
        xa = {"off8": lambda: _at_offset(xl, 8), "off1": lambda: _at_offset(xl, 1),
              "3d": lambda: xl.view(1, R, C)}.get(x, lambda: xl)()
        return (xa, w, b), [t for t in (xl, w, b) if t is not None]
    return make


def _ln_ref(x, w, b):
    return F.layer_norm(x, (x.shape[-1],), None if w is None else w.to(x.dtype), None if b is None else b.to(x.dtype),
                        LN_EPS)


@gpu
@pytest.mark.parametrize("pdt", [BF16, F32], ids=["bf16", "fp32"])
@pytest.mark.parametrize("x", ["plain", "3d", "off8"])
def test_layer_norm_kernel_path(pdt, x, env):
    R, C = 17, 256
    make = _ln_make(R, C, pdt, x=x, seed=41)
    out, (gx, gw, gb), (xa, w, b) = _fwd_bwd(lambda *a: env.F2.layer_norm(*a, LN_EPS), make, seed=7)
    _expect_kernel(env, [LN_FWD, LN_BWD])
    dy = torch.randn(out.shape, generator=_gen(7)).to(BF16).cuda().reshape(R, C)
    y64, y_terms, (dx, dxb), (dg, dgb), (db, dbb) = ln_bounds(xa.detach().reshape(R, C), w.detach(), b.detach(), dy,
                                                              LN_EPS)
    assert_within_bound(out.reshape(R, C), y64, group="layer_norm y", terms=y_terms)
    assert_within_bound(gx.reshape(R, C), dx, group="layer_norm dx", terms=[(1.0, dxb)])
    assert gw.dtype == pdt and gb.dtype == pdt
    assert_within_bound(gw, dg, group="layer_norm dgamma", terms=[(1.0, dgb)])
    assert_within_bound(gb, db, group="layer_norm dbeta", terms=[(1.0, dbb)])


LN_REFERENCE = [
    ("x-offset-2B", dict(x="off1")),
    ("fp16-params", dict(pdt=F16)),
    ("bf16-weight-fp32-bias", dict(bdt=F32)),
    ("no-affine", dict(weight=False, bias=False)),
    ("no-bias", dict(bias=False)),
    ("C-not-kernel-width", dict(C=200)),
    ("x-fp32", dict(xdt=F32, pdt=F32)),
    ("empty", dict(R=0)),
]


@gpu
@pytest.mark.parametrize("cid,kw", LN_REFERENCE, ids=[c[0] for c in LN_REFERENCE])
def test_layer_norm_reference_path(cid, kw, env):
    shape, kw = dict(R=17, C=256), dict(kw)
    shape.update({k: kw.pop(k) for k in list(kw) if k in shape})
    _expect_reference(env, lambda *a: env.F2.layer_norm(*a, LN_EPS), _ln_ref, _ln_make(**shape, **kw, seed=42))


@gpu
def test_layer_norm_wrong_length_weight_raises(env):
    _expect_raise(env, lambda *a: env.F2.layer_norm(*a, LN_EPS), _ln_ref, _ln_make(17, 256, wlen=128))


@gpu
@pytest.mark.parametrize("affine,bias", [(False, False), (True, False), (True, True)])
def test_layer_norm_module_state(affine, bias, env):
    """``nn.LayerNorm(elementwise_affine=False)`` / ``bias=False`` parameters through ``F2.layer_norm``."""
    ln = nn.LayerNorm(256, eps=LN_EPS, elementwise_affine=affine, bias=bias).cuda().to(BF16)

    def make():
        x = _randn((9, 256), 43).requires_grad_(True)
        return (x,), [x] + [p for p in ln.parameters()]
    op = lambda x: env.F2.layer_norm(x, ln.weight, ln.bias, LN_EPS)   # noqa: E731
    if affine and bias:
        _fwd_bwd(op, make, seed=8)
        _expect_kernel(env, [LN_FWD, LN_BWD])
        return
    for p in ln.parameters():
        p.grad = None
    torch.manual_seed(0)
    out, grads, _ = _fwd_bwd(op, make, seed=8)
    assert sum(env.calls.values()) == 0
    grads = [g.clone() for g in grads]
    for p in ln.parameters():
        p.grad = None
    rout, rgrads, _ = _fwd_bwd(ln, make, seed=8)
    _same(out, rout, "output")
    for g, rg in zip(grads, rgrads):
        _same(g, rg, "grad")


# ================================================================================================ dropout + add
@gpu
@pytest.mark.parametrize("case", ["offset-2B", "shape-mismatch", "fp32", "numel-not-mult-8"])
def test_dropout_add_reference_path(case, env):
    def make():
        shape = (5, 12) if case == "numel-not-mult-8" else (4, 32)
        y = _randn(shape, 51, F32 if case == "fp32" else BF16).requires_grad_(True)
        r = _randn((32,) if case == "shape-mismatch" else shape, 52, y.dtype).requires_grad_(True)
        ya = _at_offset(y, 1) if case == "offset-2B" else y
        return (ya, r), [y, r]
    _expect_reference(env, lambda y, r: env.F2.dropout_add(y, r, 0.25),
                      lambda y, r: env.F2.dropout_add_reference(y, r, 0.25), make)


@gpu
def test_dropout_add_kernel_path(env):
    """p = 1 drops everything exactly: out = residual, dy = 0, dres = dout."""
    def make():
        y = _randn((4, 32), 53).requires_grad_(True)
        r = _randn((4, 32), 54).requires_grad_(True)
        return (y, r), [y, r]
    out, (gy, gr), (y, r) = _fwd_bwd(lambda y, r: env.F2.dropout_add(y, r, 1.0), make, seed=9)
    _expect_kernel(env, ["b200dp_dropout_add"])
    _same(out, r.detach(), "p = 1: out is the residual")
    assert float(gy.abs().max()) == 0.0
    _same(gr, torch.randn(out.shape, generator=_gen(9)).to(BF16).cuda(), "dres is dout")


# ================================================================================================ BatchNorm units
def _bn(C, pdt=F32, rdt=None, momentum=0.1, affine=True, track=True, seed=0):
    bn = nn.BatchNorm2d(C, momentum=momentum, affine=affine, track_running_stats=track)
    g = _gen(seed)
    with torch.no_grad():
        if affine:
            bn.weight.copy_(torch.rand(C, generator=g) + 0.5)
            bn.bias.copy_(0.3 * torch.randn(C, generator=g))
        if track:
            bn.running_mean.copy_(0.5 * torch.randn(C, generator=g))
            bn.running_var.copy_(torch.rand(C, generator=g) + 0.5)
    bn = bn.cuda()
    for p in bn.parameters():
        p.data = p.data.to(pdt)
    if track:
        bn.running_mean.data = bn.running_mean.data.to(rdt or pdt)
        bn.running_var.data = bn.running_var.data.to(rdt or pdt)
    return bn


def _conv(Cin, Cout, k=1, stride=1, seed=0):
    conv = nn.Conv2d(Cin, Cout, k, stride, k // 2, bias=False)
    with torch.no_grad():
        conv.weight.copy_(torch.randn(conv.weight.shape, generator=_gen(seed)) / math.sqrt(Cin * k * k))
    return conv.cuda().to(BF16).to(memory_format=torch.channels_last)


def _nhwc_x(N, C, H, W, seed, dtype=BF16, cl=True):
    x = _randn((N, C, H, W), seed, dtype)
    return x.contiguous(memory_format=torch.channels_last) if cl else x


def _state(bn):
    return [t.detach().clone() for t in (bn.running_mean, bn.running_var, bn.num_batches_tracked) if t is not None]


def _torch_bn_unit(x, conv, bn, relu, residual=None):
    """What ``conv_bn_act`` means when its BatchNorm is not on the kernels: the convolution as ``ops.conv.conv2d``
    runs it (the implicit-GEMM / 1x1 GEMM kernels for bf16 NHWC, else ``F.conv2d``), then the torch module."""
    from distributed_torch_horovod_gcp_b200.ops import conv as CV
    if x.dtype == BF16 and x.is_contiguous(memory_format=torch.channels_last):
        y = bn(CV.conv2d(x, conv))
    else:
        y = bn(F.conv2d(x, conv.weight.to(x.dtype), None, conv.stride, conv.padding))
    if residual is not None:
        y = y + residual
    return F.relu(y) if relu else y


def _unit_pair(env, conv, bn, relu, residual_of, x_of, steps, train=True):
    """Runs ``F2.conv_bn_act`` on (conv, bn) and ``_torch_bn_unit`` on deep copies, ``steps`` times, each step
    with fresh seeded inputs; returns both sides' outputs, gradients and module states per step."""
    conv2, bn2 = copy.deepcopy(conv), copy.deepcopy(bn)
    bn.train(train)
    bn2.train(train)
    sides = []
    for fn, c, b in ((env.F2.conv_bn_act, conv, bn), (_torch_bn_unit, conv2, bn2)):
        steps_out = []
        for s in range(steps):
            def make():
                x = x_of(s).requires_grad_(True)
                r = residual_of(s)
                if r is not None:
                    r.requires_grad_(True)
                return (x, r), [x] + ([r] if r is not None else []) + [p for p in (c.weight, b.weight, b.bias)
                                                                       if p is not None]
            for p in (c.weight, b.weight, b.bias):
                if p is not None:
                    p.grad = None
            out, grads, args = _fwd_bwd(lambda x, r: fn(x, c, b, relu, r), make, seed=100 + s)
            steps_out.append((out, [g.clone() if g is not None else None for g in grads], _state(b), args))
        sides.append(steps_out)
    return sides


def _same_sides(sides):
    for s, (a, b) in enumerate(zip(*sides)):
        _same(a[0], b[0], f"step {s} output")
        for i, (g, rg) in enumerate(zip(a[1], b[1])):
            _same(g, rg, f"step {s} grad {i}")
        for i, (t, rt) in enumerate(zip(a[2], b[2])):
            _same(t, rt, f"step {s} BN state {i}")


BN_REFERENCE = [   # id, bn kwargs, residual form, train, x form
    ("momentum-None", dict(momentum=None), None, True, "cl"),
    ("fp16-params", dict(pdt=F16), None, True, "cl"),
    ("bf16-weight-fp32-stats", dict(pdt=BF16, rdt=F32), None, True, "cl"),
    ("fp32-weight-bf16-stats", dict(pdt=F32, rdt=BF16), None, True, "cl"),
    ("no-affine", dict(affine=False), None, True, "cl"),
    ("untracked-eval", dict(track=False), None, False, "cl"),
    ("eval-with-grad", dict(), None, False, "cl"),
    ("bcast-residual", dict(), "bcast", True, "cl"),
    ("bcast-residual-eval", dict(), "bcast", False, "cl"),
    ("fp32-residual", dict(), "fp32", True, "cl"),
    ("x-fp16", dict(), None, True, "fp16"),
    ("x-fp32-nchw", dict(), None, True, "fp32"),
    ("one-value-per-channel", dict(), None, True, "1x1"),
]


@gpu
@pytest.mark.parametrize("cid,bkw,res,train,xf", BN_REFERENCE, ids=[c[0] for c in BN_REFERENCE])
def test_conv_bn_act_reference_path(cid, bkw, res, train, xf, env):
    """Inputs the BN kernels do not take: no BN launch, and bit for bit the torch module on the convolution's
    output over 3 steps, gradients, running statistics and ``num_batches_tracked`` included.  Where torch
    raises (one value per channel in training, parameter dtypes it does not mix), the op raises the same type."""
    N, C, H, W = (1, 16, 1, 1) if xf == "1x1" else (2, 16, 5, 6)
    conv, bn = _conv(C, C, seed=61), _bn(C, seed=62, **bkw)
    dt = {"fp16": F16, "fp32": F32}.get(xf, BF16)
    x_of = lambda s: _nhwc_x(N, C, H, W, 63 + s, dt, cl=xf != "fp32")   # noqa: E731
    r_of = {None: lambda s: None, "bcast": lambda s: _randn((1, C, 1, 1), 70 + s),
            "fp32": lambda s: _nhwc_x(N, C, H, W, 70 + s, F32)}[res]
    try:
        _torch_bn_unit(x_of(0), copy.deepcopy(conv), copy.deepcopy(bn).train(train), True, r_of(0))
    except Exception as e:                   # noqa: BLE001
        with pytest.raises(type(e)):
            env.F2.conv_bn_act(x_of(0), conv, bn.train(train), True, r_of(0))
        assert env.calls[BN_FWD] == env.calls[BN_APPLY] == 0, dict(env.calls)
        return
    assert xf != "1x1", "torch accepted one value per channel in training"
    sides = _unit_pair(env, conv, bn, True, r_of, x_of, steps=3, train=train)
    assert env.calls[BN_FWD] == env.calls[BN_BWD] == env.calls[BN_APPLY] == 0, dict(env.calls)
    _same_sides(sides)
    if cid == "momentum-None":
        # the cumulative average, mom = 1 / num_batches_tracked at every step, against float64 of each batch
        from distributed_torch_horovod_gcp_b200.ops import conv as CV
        rm0, rv0 = [t.double() for t in _state(_bn(C, seed=62, **bkw))[:2]]
        for s, (out, grads, state, args) in enumerate(sides[0]):
            assert int(state[2]) == s + 1
            with torch.no_grad():
                y2 = CV.conv2d(args[0].detach(), conv).permute(0, 2, 3, 1).reshape(-1, C)
            m, var, _, Em, Evar, _ = bn_stat_bounds(y2, D=y2.shape[0])
            rm, Erm, rv, Erv = running_stats_bounds(rm0, rv0, m, var, Em, Evar, y2.shape[0], 1.0 / (s + 1), False)
            assert_within_bound(state[0], rm, group="momentum=None running_mean", terms=[(1.0, Erm)])
            assert_within_bound(state[1], rv, group="momentum=None running_var", terms=[(1.0, Erv)])
            rm0, rv0 = state[0].double(), state[1].double()


BN_KERNEL = [   # id, param dtype, residual, x form (H, W, k, stride), track_running_stats
    ("fp32-params-1x1", F32, False, (6, 5, 1, 1), True),
    ("bf16-params-residual", BF16, True, (6, 5, 1, 1), True),
    ("3x3-stride2", F32, False, (6, 8, 3, 2), True),
    ("residual-offset-2B", BF16, "offset1", (6, 5, 1, 1), True),
    ("untracked-train", BF16, False, (6, 5, 1, 1), False),
]


@gpu
@pytest.mark.parametrize("cid,pdt,res,geo,track", BN_KERNEL, ids=[c[0] for c in BN_KERNEL])
def test_conv_bn_act_kernel_path(cid, pdt, res, geo, track, env):
    """Every launch against float64 of its own inputs (the per-launch checks of the autograd module), then the
    running statistics against float64 of the batch with momentum 0.1 (untracked: batch statistics only)."""
    H, W, k, stride = geo
    N, C = 2, 16
    conv, bn = _conv(C, C, k, stride, seed=81), _bn(C, pdt, seed=82, track=track)
    OH, OW = H // stride, W // stride

    def make():
        x = _nhwc_x(N, C, H, W, 83).requires_grad_(True)
        r = rl = None
        if res:
            rl = _nhwc_x(N, C, OH, OW, 84).requires_grad_(True)
            r = (_at_offset(rl.permute(0, 2, 3, 1), 1).permute(0, 3, 1, 2) if res == "offset1" else rl)
        return (x, r), [x] + ([rl] if rl is not None else []) + [conv.weight, bn.weight, bn.bias]
    out, grads, args = _fwd_bwd(lambda x, r: env.F2.conv_bn_act(x, conv, bn, True, r), make, seed=85)
    _expect_kernel(env, [BN_FWD, BN_BWD])
    check_launches(env.spy, f"conv_bn_act {cid}")
    f = env.spy.of("bn_forward")[0]
    assert f.relu and (f.residual is None) == (not res)
    if res:
        _same(f.residual, args[1].detach().contiguous(memory_format=torch.channels_last), "BN residual is the input")
    _same(out, f.out, "output is the BN launch's")
    if not track:
        assert bn.running_mean is None and bn.num_batches_tracked is None
        return
    rm0, rv0 = [t.double() for t in _state(_bn(C, pdt, seed=82))[:2]]
    y2 = f.x.permute(0, 2, 3, 1).reshape(-1, C)
    from test_gpu_autograd_numerics import bn_forward_of   # the statistics depth of this launch's source
    D = bn_forward_of(env.spy, f).D
    m, var, _, Em, Evar, _ = bn_stat_bounds(y2, D)
    rm, Erm, rv, Erv = running_stats_bounds(rm0, rv0, m, var, Em, Evar, y2.shape[0], 0.1, pdt == BF16)
    assert_within_bound(bn.running_mean, rm, group="conv_bn_act running_mean", terms=[(1.0, Erm)])
    assert_within_bound(bn.running_var, rv, group="conv_bn_act running_var", terms=[(1.0, Erv)])
    assert int(bn.num_batches_tracked) == 1


@gpu
def test_conv_bn_act_eval_kernel_path(env):
    """Eval mode with running statistics: the fused apply pass; ``test_bn_inference_apply_vs_fp64`` bounds it."""
    conv, bn = _conv(16, 16, seed=91), _bn(16, seed=92)
    bn.eval()
    with torch.no_grad():
        env.F2.conv_bn_act(_nhwc_x(2, 16, 4, 4, 93), conv, bn, True)
    _expect_kernel(env, [BN_APPLY])


# ================================================================================================ ResNet blocks
def _block(kind, **bkw):
    from distributed_torch_horovod_gcp_b200.models.resnet import BasicBlock, Bottleneck
    torch.manual_seed(5)
    if kind == "basic":
        blk = BasicBlock(16, 16)
    else:
        ds = nn.Sequential(nn.Conv2d(32, 64, 1, 2, bias=False), nn.BatchNorm2d(64))
        blk = Bottleneck(32, 16, stride=2, downsample=ds)
    blk = blk.cuda().to(BF16).to(memory_format=torch.channels_last)
    for m in blk.modules():
        if isinstance(m, nn.BatchNorm2d):
            for k, v in bkw.items():
                if k == "momentum":
                    m.momentum = v
                elif k == "pdt":
                    for p in m.parameters():
                        p.data = p.data.to(v)
                    m.running_mean.data = m.running_mean.data.to(v)
                    m.running_var.data = m.running_var.data.to(v)
    return blk


def _reference_block(blk, x):
    if hasattr(blk, "conv3"):
        out = _torch_bn_unit(x, blk.conv1, blk.bn1, True)
        out = _torch_bn_unit(out, blk.conv2, blk.bn2, True)
        idn = _torch_bn_unit(x, blk.downsample[0], blk.downsample[1], False)
        return _torch_bn_unit(out, blk.conv3, blk.bn3, True, idn)
    out = _torch_bn_unit(x, blk.conv1, blk.bn1, True)
    return _torch_bn_unit(out, blk.conv2, blk.bn2, True, x)


BLOCK_CASES = [   # id, kind, bn kwargs, mode (train / eval / eval-no-grad), kernel?
    ("basic-train", "basic", dict(), "train", True),
    ("bottleneck-train", "bottleneck", dict(), "train", True),
    ("bottleneck-momentum-None", "bottleneck", dict(momentum=None), "train", False),
    ("basic-momentum-None", "basic", dict(momentum=None), "train", False),
    ("bottleneck-fp16-bn", "bottleneck", dict(pdt=F16), "train", False),
    ("bottleneck-eval-with-grad", "bottleneck", dict(), "eval", False),
    ("bottleneck-eval-no-grad", "bottleneck", dict(), "eval-no-grad", True),
]


@gpu
@pytest.mark.parametrize("cid,kind,bkw,mode,kernel", BLOCK_CASES, ids=[c[0] for c in BLOCK_CASES])
def test_resnet_block_dispatch(cid, kind, bkw, mode, kernel, env):
    blk = _block(kind, **bkw).train(mode == "train")
    ref = copy.deepcopy(blk)
    Cin = 16 if kind == "basic" else 32

    def run(b, fn):
        for p in b.parameters():
            p.grad = None

        def make():
            x = _nhwc_x(3, Cin, 6, 6, 101).requires_grad_(True)
            return (x,), [x] + list(b.parameters())
        if mode == "eval-no-grad":
            with torch.no_grad():
                return _fwd_bwd(fn, make, seed=102)
        return _fwd_bwd(fn, make, seed=102)
    try:
        rout, rgrads, _ = run(ref, lambda x: _reference_block(ref, x))
    except Exception as e:                   # noqa: BLE001
        with pytest.raises(type(e)):
            run(blk, blk)
        assert env.calls[BN_FWD] == env.calls[BN_APPLY] == 0, dict(env.calls)
        return
    env.calls.clear()
    env.spy.calls.clear()
    out, grads, _ = run(blk, blk)
    if kernel and mode == "train":
        _expect_kernel(env, [BN_FWD, BN_BWD] + ([GEMM] if kind == "bottleneck" else ["b200dp_conv_fprop"]))
        check_launches(env.spy, f"block {cid}")
        _same(out, env.spy.of("bn_forward")[-1].out, "block output is the last BN launch's")
        return
    if kernel:
        _expect_kernel(env, [BN_APPLY])
        return
    assert env.calls[BN_FWD] == env.calls[BN_APPLY] == 0, dict(env.calls)
    _same(out, rout, "block output")
    for i, (g, rg) in enumerate(zip(grads, rgrads)):
        _same(g, rg, f"block grad {i}")
    for (n, t), (_, rt) in zip(blk.named_buffers(), ref.named_buffers()):
        _same(t, rt, n)


# ================================================================================================ pooling
@gpu
@pytest.mark.parametrize("case,kernel", [("C16-odd-HW", True), ("C12", False), ("fp32", False), ("nchw", False),
                                         ("offset-2B", False)])
def test_pools_dispatch(case, kernel, env):
    N, C, H, W = 2, (12 if case == "C12" else 16), 7, 9

    def make():
        x = _nhwc_x(N, C, H, W, 111, F32 if case == "fp32" else BF16, cl=case != "nchw").requires_grad_(True)
        xa = _at_offset(x.permute(0, 2, 3, 1), 1).permute(0, 3, 1, 2) if case == "offset-2B" else x
        return (xa,), [x]
    refs = {"max_pool_3x3_s2": lambda x: F.max_pool2d(x, 3, 2, 1), "global_avg_pool": lambda x: x.mean(dim=(2, 3))}
    for name, ref in refs.items():
        env.calls.clear()
        op = getattr(env.F2, name)
        if not kernel:
            _expect_reference(env, op, ref, make)
            continue
        out, (gx,), (x,) = _fwd_bwd(op, make, seed=112)
        _expect_kernel(env, ["b200dp_maxpool_fwd", "b200dp_maxpool_bwd"] if name.startswith("max") else
                       ["b200dp_avgpool_fwd", "b200dp_avgpool_bwd"])
        if name.startswith("max"):
            _same(out, ref(x.detach()), "max-pool is exact")     # a max of bf16 values is one of them
            # every output gradient lands on one input of its window: the totals agree within the bf16 stores
            dy = torch.randn(out.shape, generator=_gen(112)).to(BF16).cuda().double()
            tot = dy.sum(dim=(2, 3))
            assert_within_bound(gx.double().sum(dim=(2, 3)), tot, group="max-pool dx total",
                                terms=[(2 ** -8 * 1.01, dy.abs().sum(dim=(2, 3)))])
        else:
            ref64 = x.detach().double().mean(dim=(2, 3))
            E = 2 * H * W * U32 * x.detach().double().abs().mean(dim=(2, 3))
            assert_within_bound(out, ref64, group="avg-pool y", terms=[(1.0, bf16_store(E, ref64))])


# ================================================================================================ patch embed + LM head
@gpu
@pytest.mark.parametrize("bdt,kernel", [(F32, True), (F16, False)], ids=["fp32-bias", "fp16-bias"])
def test_patch_embed_dispatch(bdt, kernel, env):
    B, P, D = 2, 4, 32

    def make():
        x = _randn((B, 3, 8, 12), 121).requires_grad_(True)
        w = _randn((D, 3, P, P), 122, BF16, 0.2).requires_grad_(True)
        b = _randn((D,), 123, bdt).requires_grad_(True)
        return (x, w, b), [x, w, b]
    op = lambda x, w, b: env.F2.patch_embed(x, w, b, P)   # noqa: E731
    ref = lambda x, w, b: F.conv2d(x, w, b.to(x.dtype), stride=P).flatten(2).transpose(1, 2)   # noqa: E731
    if not kernel:
        _expect_reference(env, op, lambda x, w, b: env.F2.linear_reference(
            x.reshape(B, 3, 2, P, 3, P).permute(0, 2, 4, 1, 3, 5).reshape(B, 6, 3 * P * P), w.reshape(D, -1), b), make)
        return
    out, grads, (x, w, b) = _fwd_bwd(op, make, seed=124)
    _expect_kernel(env, [GEMM])
    check_launches(env.spy, "patch_embed")
    cols = x.detach().reshape(B, 3, 2, P, 3, P).permute(0, 2, 4, 1, 3, 5).reshape(B * 6, 3 * P * P)
    (y, E), _ = epilogue_bounds(cols, w.detach().reshape(D, -1), 1.0, b.detach())
    assert_within_bound(out.reshape(-1, D), y, group="patch_embed y", terms=[(1.0, E)])
    assert ref(x.detach(), w.detach(), b.detach()).shape == out.shape


@gpu
@pytest.mark.parametrize("case,kernel", [("V-mult-8", True), ("V-not-mult-8", False), ("x-fp32", False),
                                         ("weight-transposed", False)])
def test_linear_cross_entropy_dispatch(case, kernel, env):
    N, D = 37, 64
    V = 100 if case == "V-not-mult-8" else 96

    def make():
        x = _randn((N, D), 131, F32 if case == "x-fp32" else BF16).requires_grad_(True)
        wl = _randn((D, V) if case == "weight-transposed" else (V, D), 132, BF16, 0.3).requires_grad_(True)
        t = torch.randint(0, V, (N,), generator=_gen(133)).cuda()
        return (x, wl.t() if case == "weight-transposed" else wl, t), [x, wl]
    op, ref = env.F2.linear_cross_entropy, env.F2.linear_cross_entropy_reference
    if case == "x-fp32":              # torch's F.linear refuses an fp32 x against a bf16 weight
        _expect_raise(env, lambda x, w, t: op(x, w, t, reduction="none"),
                      lambda x, w, t: ref(x, w, t, reduction="none"), make)
        return
    if not kernel:
        _expect_reference(env, lambda x, w, t: op(x, w, t, reduction="none"),
                          lambda x, w, t: ref(x, w, t, reduction="none"), make)
        return
    out, grads, (x, w, t) = _fwd_bwd(lambda x, w, t: op(x, w, t, reduction="none"), make, seed=134)
    _expect_kernel(env, ["b200dp_xent_fwd", "b200dp_xent_grad", GEMM])
    loss64, bound = xent_fwd_bounds(x.detach(), w.detach(), t)
    assert_within_bound(out, loss64, group="linear_cross_entropy loss", terms=[(1.0, bound)])
    assert all(g is not None and bool(torch.isfinite(g.float()).all()) for g in grads)


# ================================================================================================ guard self-tests (CPU)
def _gemm_args(A=0x1000, B=0x3000, C=0x5000, M=4, N=8, K=8, residual=None, preact=None, bias_bf16=None):
    return (A, B, C, M, N, K, K, K, N, 0, 0, bias_bf16, None, residual, preact, 0, 0, 1, 1.0, 1, 0, 0, None, None, 0)


# three 256-byte blocks, the second and third back to back
BLOCKS = [(0x1000, 0x1100), (0x3000, 0x3100), (0x3100, 0x3200), (0x5000, 0x5100)]


def test_guard_accepts_valid_launches():
    launch_guard.check("b200dp_gemm_bf16", _gemm_args(), BLOCKS)
    launch_guard.check("b200dp_gemm_bf16", _gemm_args(residual=0x3100, preact=0x3104, bias_bf16=0x50f0), BLOCKS)
    # an extent that ends exactly at its block's end: A is [4, 8] bf16 = 64 bytes at 0x10c0
    launch_guard.check("b200dp_gemm_bf16", _gemm_args(A=0x10c0), BLOCKS)
    launch_guard.check("b200dp_ln_fwd", (0x3000, 0x3100, 0x1000, 0x1080, 0x5000, 0x5010, 1, 64, 1e-6, 1, 0),
                       BLOCKS)


@pytest.mark.parametrize("case", ["misaligned-A", "misaligned-residual", "misaligned-preact", "past-end",
                                  "spans-two-blocks", "no-allocation", "null-required", "relu-mask-null",
                                  "unknown-symbol", "arity"])
def test_guard_rejects_each_violation(case):
    sym, args = "b200dp_gemm_bf16", _gemm_args()
    if case == "misaligned-A":
        args = _gemm_args(A=0x1008)
    elif case == "misaligned-residual":
        args = _gemm_args(residual=0x3102)
    elif case == "misaligned-preact":
        args = _gemm_args(preact=0x3102)
    elif case == "past-end":
        args = _gemm_args(A=0x10c2 + 14)        # 16-byte aligned 0x10d0: 64 bytes end 16 past 0x1100
    elif case == "spans-two-blocks":
        args = _gemm_args(B=0x30d0)            # [8, 8] bf16 = 128 bytes from 0x30d0 runs into the next block
    elif case == "no-allocation":
        args = _gemm_args(C=0x7000)
    elif case == "null-required":
        args = _gemm_args(B=None)
    elif case == "relu-mask-null":
        sym = "b200dp_bn_bwd"
        args = (0x3000, 0x3000, None, 0x5000, None, 0x1000, 0x1000, 0x1000, 0x1000, None, None, 0, 1, 8, 1, 0)
    elif case == "unknown-symbol":
        sym = "b200dp_not_a_kernel"
    else:
        args = args[:-1]
    with pytest.raises(GuardError):
        launch_guard.check(sym, args, BLOCKS)


def test_guard_tightest_extent():
    """The largest extent that fits is accepted; one element more is rejected."""
    # bn_apply: x, res, y are 2 M C bytes; with C = 8, M = 16 rows fill 256 bytes exactly
    ok = (0x3000, None, 0x5000, 0x1000, 0x1080, 16, 8, 0, 0)
    launch_guard.check("b200dp_bn_apply", ok, BLOCKS)
    with pytest.raises(GuardError):
        launch_guard.check("b200dp_bn_apply", ok[:5] + (17,) + ok[6:], BLOCKS)


def test_guarded_lib_forwards_counts_and_refuses():
    class Fake:
        def __init__(self):
            self.got = []

        def b200dp_bn_apply(self, *a):
            self.got.append(a)
            return 0

        def b200dp_bn_supported(self, C):
            return 1

        def b200dp_secret_launch(self, *a):
            raise AssertionError("must not be reached")

    from collections import Counter
    fake, calls = Fake(), Counter()
    lib = launch_guard.GuardedLib(fake, calls, blocks=lambda: BLOCKS)
    assert lib.b200dp_bn_supported(8) == 1
    assert lib.b200dp_bn_apply(0x3000, None, 0x5000, 0x1000, 0x1080, 16, 8, 0, 0) == 0
    assert calls["b200dp_bn_apply"] == 1 and len(fake.got) == 1
    with pytest.raises(GuardError):
        lib.b200dp_bn_apply(0x3008, None, 0x5000, 0x1000, 0x1080, 16, 8, 0, 0)
    assert calls["b200dp_bn_apply"] == 1 and len(fake.got) == 1
    with pytest.raises(GuardError):
        lib.b200dp_secret_launch(1)
    assert not hasattr(lib, "b200dp_missing")
