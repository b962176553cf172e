"""The autograd nodes of the kernel path against float64, one launch at a time: ``_LinearFn``, ``_MLPFn``,
``_QKVFn``, ``wgrad`` and ``bias_grad`` (ops/gemm.py), ``_BottleneckFn`` (ops/bottleneck.py), ``_ConvFn``
(ops/conv.py), ``_BNActFn`` (ops/bn.py) and the weight gradients written straight into gradient-bucket slots
(ops/grad_sink.py).

The kernels are bounded element by element in ``test_gpu_resnet_numerics.py`` and ``test_gpu_reductions.py``.  What
those tests cannot see is the glue between launches: which saved tensor feeds which launch, operand majorness and
row strides, the split count ``_splits_for`` picks and the store mode that follows from it, the PyTorch code run
between launches, and accumulation into a bucket slot on later backward passes.  Here spies on the module
attributes the nodes call (``ops.gemm.gemm``; ``ops.conv.conv_fprop`` / ``conv_dgrad`` / ``conv_wgrad``;
``ops.bn.bn_forward`` / ``bn_backward``) record every launch's inputs and output, and

1. every launch is bounded against float64 of its own recorded inputs, with the bound helpers of the kernel tests
   (``epilogue_bounds``, ``conv_bound``, ``bn_fwd_bounds``, ``bn_bwd_bounds``); a freshly allocated GEMM output is
   filled with NaN before the launch, so an element no kernel writes fails;
2. every hand-off is checked bit for bit: each launch reads the tensors the node is meant to feed it, and every
   returned ``.grad`` is the last launch's output, or that after its one documented conversion;
3. for ``linear``, ``mlp`` and ``qkv_proj``, dx / dW / db are also bounded against float64 of the whole node on its
   exact inputs, each stage's bound propagated through the next (nothing is fitted to observed errors).

The PyTorch code between launches has bounds of its own: ``act_backward_bound``, the ``acc[:, 0].to(dtype)`` of
``bias_grad`` and ``accumulate_bound`` for a bucket slot's ``fl(prev + dW)``.  The CPU tests at the end check them,
and the QKV ``dx`` chain, against fp32 emulations, and that moving the tightest element to 1.01x its bound fails.
"""
import math
import os
import sys
from types import SimpleNamespace

import pytest
import torch
import torch.nn as nn

TESTS = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(TESTS)
for _p in (ROOT, TESTS):
    if _p not in sys.path:
        sys.path.insert(0, _p)

import fp64_bounds  # noqa: E402
from fp64_bounds import U32, U_BF16, assert_within_bound, report_ratios  # noqa: E402
from test_gpu_reductions import _wgrad_ref  # noqa: E402
from test_gpu_resnet_numerics import (FLUSH, _bits_to_mask, _gelu_grad64, _pad64, _sms, _to2, bf16_store,  # noqa: E402
                                      bn_bwd_bounds, bn_fwd_bounds, conv_bound, conv_dgrad_ref, conv_fprop_ref,
                                      epilogue_bounds, standalone_depth, stats_depth)

gpu = pytest.mark.gpu
BF16, F32 = torch.bfloat16, torch.float32

# Accuracy of the CUDA fp32 library functions PyTorch's erf / exp call (CUDA C Programming Guide, "Single-Precision
# Mathematical Functions": erff and expf, 2 ulp each); 1 ulp <= 2u relative.
U_ERFF = 4 * U32
U_EXPF = 4 * U32
GELU2_MAX = 0.8          # max |gelu''(z)| = 2 phi(0) = 0.7979: how far gelu' moves when z does


@pytest.fixture(scope="module", autouse=True)
def _report_ratios():
    yield
    report_ratios()


def _check(out, ref, bound, group):
    assert_within_bound(out, ref, group=group, terms=[(1.0, bound)])


def _bits(t):
    return t.detach().contiguous().view({BF16: torch.int16, F32: torch.int32, torch.uint8: torch.uint8}[t.dtype])


def same_ptr(a, b):
    return a is not None and b is not None and a.data_ptr() == b.data_ptr()


def same_bits(a, b, what):
    assert a.shape == b.shape and a.dtype == b.dtype, f"{what}: {a.shape}/{a.dtype} vs {b.shape}/{b.dtype}"
    assert torch.equal(_bits(a), _bits(b)), f"{what}: bits differ"


def _ops():
    from distributed_torch_horovod_gcp_b200.ops import bn, bottleneck, conv, gemm, grad_sink, kernels
    assert kernels.has("gemm") and kernels.has("conv_implicit_gemm") and kernels.has("conv_bn_act"), \
        "libb200dp_kernels.so not loaded"
    return SimpleNamespace(gemm=gemm, conv=conv, bn=bn, bottleneck=bottleneck, grad_sink=grad_sink)


# ================================================================================================ spies
class Spy:
    """Wraps the kernel entry points the autograd nodes reach through their module globals.  Each wrapper calls
    through and appends a record of its inputs and output to ``calls``, in launch order.  Inputs a launch may
    overwrite (an aliased residual, an accumulated destination) are cloned before it; outputs are cloned after."""

    def __init__(self, monkeypatch, ops):
        self.calls = []
        self.ops = ops
        g, c, b = ops.gemm, ops.conv, ops.bn
        for mod, name, wrap in ((g, "gemm", self._gemm), (c, "conv_fprop", self._conv_fprop),
                                (c, "conv_dgrad", self._conv_dgrad), (c, "conv_wgrad", self._conv_wgrad),
                                (b, "bn_forward", self._bn_forward), (b, "bn_backward", self._bn_backward)):
            monkeypatch.setattr(mod, name, wrap(getattr(mod, name)))

    def of(self, op):
        return [r for r in self.calls if r.op == op]

    def _gemm(self, f):
        def gemm(a, b, out, M, N, K, *, a_mn=False, b_mn=False, bias=None, residual=None, preact=None, act=0,
                 out_mode=0, alpha=1.0, splits=1, block_n=0, max_ctas=0, stats=None, res_mask=None):
            alias = residual is not None and residual.data_ptr() == out.data_ptr()
            r = SimpleNamespace(op="gemm", a=a, b=b, M=M, N=N, K=K, a_mn=a_mn, b_mn=b_mn, bias=bias, act=act,
                                residual=residual.clone() if alias else residual, alias=alias, out_mode=out_mode,
                                alpha=alpha, splits=splits, stats=stats, res_mask=res_mask, out_ptr=out.data_ptr(),
                                prev=out.clone() if out_mode == 1 else None)
            if out_mode != 1 and not alias:
                out.fill_(float("nan"))
            if preact is not None:
                preact.fill_(float("nan"))
            f(a, b, out, M, N, K, a_mn=a_mn, b_mn=b_mn, bias=bias, residual=residual, preact=preact, act=act,
              out_mode=out_mode, alpha=alpha, splits=splits, block_n=block_n, max_ctas=max_ctas, stats=stats,
              res_mask=res_mask)
            r.out, r.out_t, r.preact = out.clone(), out, preact.clone() if preact is not None else None
            self.calls.append(r)
            return out
        return gemm

    def _conv_fprop(self, f):
        def conv_fprop(x, w, stride, pad, stats=None):
            y = f(x, w, stride, pad, stats)
            self.calls.append(SimpleNamespace(op="conv_fprop", x=x, w=w, stride=stride, pad=pad, stats=stats,
                                              out=y.clone(memory_format=torch.channels_last), out_t=y))
            return y
        return conv_fprop

    def _conv_dgrad(self, f):
        def conv_dgrad(dy, w, x_shape, stride, pad):
            dx = f(dy, w, x_shape, stride, pad)
            self.calls.append(SimpleNamespace(op="conv_dgrad", dy=dy, w=w, x_shape=tuple(x_shape), stride=stride,
                                              pad=pad, out=dx.clone(memory_format=torch.channels_last)))
            return dx
        return conv_dgrad

    def _conv_wgrad(self, f):
        def conv_wgrad(dy, x, weight, stride, pad):
            dst, acc, _ = self.ops.grad_sink.begin(weight, krsc=True)
            prev = dst.clone(memory_format=torch.channels_last) if acc else None
            ret = f(dy, x, weight, stride, pad)
            out = ret if ret is not None else weight.grad
            self.calls.append(SimpleNamespace(op="conv_wgrad", dy=dy, x=x, weight=weight, stride=stride, pad=pad,
                                              sink=dst is not None, prev=prev, returned=ret is not None,
                                              out=out.clone(memory_format=torch.channels_last)))
            return ret
        return conv_wgrad

    def _bn_forward(self, f):
        def bn_forward(x, bn, residual, relu, stats_in=None, grads=(True, True)):
            y, mask, ws = f(x, bn, residual, relu, stats_in, grads)
            self.calls.append(SimpleNamespace(op="bn_forward", x=x, bn=bn, residual=residual, relu=relu,
                                              stats=stats_in, out=y.clone(memory_format=torch.channels_last), out_t=y,
                                              mask=mask, ws=ws, gamma=bn.weight.detach().clone(),
                                              beta=bn.bias.detach().clone()))
            return y, mask, ws
        return bn_forward

    def _bn_backward(self, f):
        def bn_backward(dy, bn, x, mask, ws, write_dres=False):
            dx, dg, db, dres = f(dy, bn, x, mask, ws, write_dres)
            r = SimpleNamespace(op="bn_backward", dy=dy, bn=bn, x=x, mask=mask, ws=ws, write_dres=write_dres,
                                out=dx.clone(memory_format=torch.channels_last), out_t=dx, direct=dg is None,
                                dres=dres.clone(memory_format=torch.channels_last) if dres is not None else None)
            r.dg = (dg if dg is not None else bn.weight.grad).clone()
            r.db = (db if db is not None else bn.bias.grad).clone()
            self.calls.append(r)
            return dx, dg, db, dres
        return bn_backward


# ================================================================================================ per-launch bounds
def gemm_operands(r):
    """The logical A [M, K] and B [N, K] a recorded launch read."""
    A = r.a.t() if r.a_mn else r.a
    B = r.b.t() if r.b_mn else r.b
    assert tuple(A.shape) == (r.M, r.K) and tuple(B.shape) == (r.N, r.K), (A.shape, B.shape, r.M, r.N, r.K)
    return A, B


def gemm_role(r):
    if r.a_mn and r.b_mn:
        return "bias_grad" if r.N == 8 and r.out.dtype == F32 and r.out_mode == 1 else "wgrad"
    if r.b_mn:
        return "dgrad act3" if r.act == 3 else "dgrad"
    return "fwd"


def check_gemm(r, tag):
    """The launch against float64 of its recorded inputs; returns the reference and bound of its output."""
    A, B = gemm_operands(r)
    res = r.prev if r.out_mode == 1 else r.residual
    if r.res_mask is not None:
        res = res * _bits_to_mask(r.res_mask, r.M, r.N).to(res.dtype)
    (y, E), (z, Ez) = epilogue_bounds(A, B, r.alpha, r.bias, r.act, res, out_fp32=r.out.dtype == F32)
    group = f"{tag} gemm {gemm_role(r)}"
    _check(r.out, y, E, group)
    if r.preact is not None:
        _check(r.preact, z, Ez, f"{tag} gemm fwd preact")
    return y, E


def check_conv(r, tag):
    if r.op == "conv_fprop":
        R, Cin = r.w.shape[2], r.w.shape[1]
        y64, ym = conv_fprop_ref(r.x, r.w, r.stride, r.pad)
        _check(r.out, y64, conv_bound(y64, ym, R * R * _pad64(Cin)), f"{tag} conv fprop")
    elif r.op == "conv_dgrad":
        R, Cout = r.w.shape[2], r.w.shape[0]
        dx64, dxm = conv_dgrad_ref(r.dy, r.w, r.x_shape, r.stride, r.pad)
        _check(r.out, dx64, conv_bound(dx64, dxm, R * R * _pad64(Cout)), f"{tag} conv dgrad")
    else:
        ref, E = conv_wgrad_ref(r)
        _check(r.out.permute(0, 2, 3, 1), ref, bf16_store(E, ref), f"{tag} conv wgrad")


def conv_wgrad_ref(r):
    """float64 dW [Cout][R][S][Cin] of a recorded conv_wgrad (+ the slot's previous value when it accumulated) and
    the bound of its fp32 sum before the one store: 2 n u sum|terms| over n = pixels (+ 1 for the add)."""
    R = r.weight.shape[2]
    ref, mag = _wgrad_ref(r.x, r.dy, R, r.stride, r.pad)
    n = _pad64(r.dy.shape[0] * r.dy.shape[2] * r.dy.shape[3])
    if r.prev is not None:
        p = r.prev.permute(0, 2, 3, 1).double()
        return ref + p, 2 * (n + 1) * U32 * (mag + p.abs())
    return ref, 2 * n * U32 * mag


def _stats_src(spy, r):
    """Which launch accumulated the statistics a bn_forward read: 'gemm', 'conv' or 'standalone'."""
    if r.stats is None:
        return "standalone"
    i = spy.calls.index(r)
    for p in reversed(spy.calls[:i]):
        if p.op in ("gemm", "conv_fprop") and p.stats is not None and p.stats.data_ptr() == r.stats.data_ptr():
            return "gemm" if p.op == "gemm" else "conv"
    raise AssertionError("bn_forward read a statistics buffer no launch filled")


def check_bn_forward(spy, r, tag):
    N, C, H, W = r.x.shape
    r.D = stats_depth(_stats_src(spy, r), N, C, H, W)
    res2 = _to2(r.residual) if r.residual is not None else None
    yr, yb, pre, Epre = bn_fwd_bounds(_to2(r.x), r.gamma, r.beta, res2, r.relu, r.D)
    _check(_to2(r.out), yr, yb, f"{tag} bn fwd")
    if r.relu:
        bits = _bits_to_mask(r.mask, N * H * W, C)
        sure = pre.abs() > Epre
        assert bool((bits[sure] == (pre[sure] > 0)).all()), "ReLU mask bit disagrees with the sign of y"
        assert bool((_to2(r.out)[~bits] == 0).all()), "y nonzero where the mask bit is clear"


def bn_forward_of(spy, r):
    """The bn_forward whose saved (mean, invstd, a) a bn_backward read."""
    for f in spy.of("bn_forward"):
        if f.ws[0].data_ptr() == r.ws[0].data_ptr():
            assert all(a.data_ptr() == b.data_ptr() for a, b in zip(f.ws, r.ws))
            return f
    raise AssertionError("bn_backward read statistics no bn_forward wrote")


def bn_dz2(r):
    N, C, H, W = r.x.shape
    dy2 = _to2(r.dy)
    if r.mask is None:
        return dy2
    return dy2 * _bits_to_mask(r.mask, N * H * W, C).to(BF16)


def check_bn_backward(spy, r, tag):
    f = bn_forward_of(spy, r)
    same_bits(r.x, f.x, "bn_backward reads the input its forward normalised")
    N, C, H, W = r.x.shape
    M = N * H * W
    dz2 = bn_dz2(r)
    pbf16 = r.bn.weight.dtype == BF16
    (dxr, dxb), (dgr, dgb), (dbr, dbb) = bn_bwd_bounds(_to2(r.x), dz2, f.gamma, f.D, standalone_depth(M, C, _sms()),
                                                       pbf16)
    _check(_to2(r.out), dxr, dxb, f"{tag} bn bwd dx")
    _check(r.dg, dgr, dgb, f"{tag} bn bwd dgamma")
    _check(r.db, dbr, dbb, f"{tag} bn bwd dbeta")
    if r.dres is not None:
        assert torch.equal(_to2(r.dres), dz2), "dres is not the masked dy"
    return (dgr, dgb), (dbr, dbb)


def check_launches(spy, tag):
    """Every recorded launch against float64 of its own inputs."""
    for r in spy.calls:
        if r.op == "gemm":
            check_gemm(r, tag)
        elif r.op.startswith("conv"):
            check_conv(r, tag)
        elif r.op == "bn_forward":
            check_bn_forward(spy, r, tag)
        else:
            check_bn_backward(spy, r, tag)


# ================================================================================================ glue bounds
def act_backward_bound(dy, z, act):
    """float64 dy * act'(z) and the bound of ``act_backward(dy, z, act)`` (z: the bf16 tensor it reads).
    ReLU: dy * (z > 0) in bf16 is exact.  GELU, in fp32:
    - cdf = 0.5 fl(1 + erff(fl(z c~))), c~ = fp32(1/sqrt 2): the constant and the product move the argument by
      2.02 u |z c| (|erf'| <= 2/sqrt(pi)), erff adds U_ERFF |erf|, the sum one rounding: E_cdf = 0.5 (E_e + u (|1 + erf|
      + E_e)); the 0.5 is exact;
    - pdf = fl(c2~ expf(fl(fl(-0.5 z) z))): the rounded square moves exp by u z^2/2 relative, expf adds U_EXPF, the
      fp32 constant and the product 2u: E_pdf = 1.01 (u z^2 / 2 + U_EXPF + 2u) pdf;
    - g = fl(cdf + fl(z pdf)): E_g = (E_cdf + |z| E_pdf)(1 + 2.02 u) + 2.02 u (|cdf| + |z| pdf);
    - fl(dy g): |dy| E_g + u |dy| (|g| + E_g), then the bf16 store."""
    d, a = dy.double(), z.double()
    if act == 1:
        return d * (a > 0).double(), torch.zeros_like(d)
    c = 1 / math.sqrt(2.0)
    erf = torch.erf(a * c)
    Ee = U_ERFF * erf.abs() + 2.02 * U32 * (a * c).abs() * (2 / math.sqrt(math.pi))
    cdf = 0.5 * (1 + erf)
    Ecdf = 0.5 * (Ee + U32 * ((1 + erf).abs() + Ee))
    pdf = torch.exp(-0.5 * a * a) / math.sqrt(2 * math.pi)
    Epdf = 1.01 * (U32 * a * a / 2 + U_EXPF + 2 * U32) * pdf
    g = cdf + a * pdf
    Eg = (Ecdf + a.abs() * Epdf) * (1 + 2.02 * U32) + 2.02 * U32 * (cdf.abs() + a.abs() * pdf)
    v = d * g
    E = d.abs() * Eg + U32 * d.abs() * (g.abs() + Eg)
    return v, bf16_store(E, v)


def bias_grad_bound(y, E, dtype):
    """``acc[:, 0].to(dtype)``: the fp32 column (within E of y) kept as it is, or rounded once to bf16."""
    return bf16_store(E, y) if dtype == BF16 else E


def accumulate_bound(prev, ref, E1):
    """A bucket slot after ``fl(prev + dW)``: ``ref`` the float64 dW of this pass, ``E1`` its bound as one bf16
    value.  Autograd's AccumulateGrad adds that bf16 dW and rounds once more; the kernels add their fp32 sum and
    round once, which has one rounding fewer.  Both: |slot - (prev + ref)| <= bf16_store(E1, prev + ref)."""
    return bf16_store(E1, prev.double() + ref)


def prop_gemm(EA, A, B, K):
    """Bound of an fp32-accumulated C = A B^T (A [M, K] with elementwise error EA against A*, B exact) against
    A* B^T, before the store: EA |B|^T + 2 pad64(K) u |A| |B|^T (|A| the values the GEMM read)."""
    Bd = B.double().abs()
    return EA @ Bd.t() + 2 * _pad64(K) * U32 * (A.double().abs() @ Bd.t())


def qkv_dx_bound(gs, ws):
    """dx = bf16(bf16(bf16(dq Wq) + dk Wk) + dv Wv): three fp32 accumulations, each previous partial read exactly
    as the epilogue residual, three bf16 stores.  Returns float64 dq Wq + dk Wk + dv Wv and its bound."""
    S = E = None
    for g, w in zip(gs, ws):
        P = g.double() @ w.double()
        Ea = 2 * _pad64(g.shape[1]) * U32 * (g.double().abs() @ w.double().abs())
        if S is None:
            S, E = P, bf16_store(Ea, P)
        else:
            S = S + P
            Ein = Ea + E
            E = bf16_store(Ein + U32 * (S.abs() + Ein), S)
    return S, E


# ================================================================================================ linear
def _x_form(form, M, K, gen):
    """A leaf and the view ``linear`` gets: 2-D, 3-D, the first token of [M, 197, K] (strided rows the node keeps
    without a copy) or the first K columns of [M, K + 1] (an odd row stride: the node copies)."""
    if form == "strided":
        leaf = torch.randn(M, 197, K, device="cuda", generator=gen).to(BF16)
        return leaf, lambda t: t[:, 0]
    if form == "copy":
        leaf = torch.randn(M, K + 1, device="cuda", generator=gen).to(BF16)
        return leaf, lambda t: t[:, :K]
    leaf = torch.randn(M, K, device="cuda", generator=gen).to(BF16)
    if form == "3d":
        d = 2 if M % 2 == 0 else 1
        return leaf, lambda t: t.view(d, M // d, K)
    return leaf, lambda t: t


ACTS = {None: 0, "relu": 1, "gelu": 2}


def run_linear(M, N, K, act, bdt, with_res, form, need, seed, spy, ops):
    """``linear`` forward and backward with spies; ``need`` the subset of {x, w, b, res} that requires grad.
    Checks every launch, every hand-off and the end-to-end bounds; returns the wgrad split count."""
    gen = torch.Generator(device="cuda").manual_seed(seed)
    xl, view = _x_form(form, M, K, gen)
    # GELU: pre-activations over about +-8, the erf tails included
    scale = 2.5 if act == "gelu" else 1.0
    w = (torch.randn(N, K, device="cuda", generator=gen) * scale / math.sqrt(K)).to(BF16)
    b = (torch.randn(N, device="cuda", generator=gen)).to(bdt) if bdt is not None else None
    res = torch.randn(M, N, device="cuda", generator=gen).to(BF16) if with_res else None
    dy = torch.randn(M, N, device="cuda", generator=gen).to(BF16)
    for t, k in ((xl, "x"), (w, "w"), (b, "b"), (res, "res")):
        if t is not None:
            t.requires_grad_(k in need)
    x = view(xl)
    r_in = res.view(*x.shape[:-1], N) if res is not None else None
    y = ops.gemm.linear(x, w, b, act, r_in)
    y.backward(dy.view(y.shape))
    torch.cuda.synchronize()
    with torch.no_grad():
        return _check_linear(spy, ops, M, N, K, act, bdt, form, need, xl, view, w, b, res, dy, y)


def _check_linear(spy, ops, M, N, K, act, bdt, form, need, xl, view, w, b, res, dy, y):
    calls = spy.of("gemm")
    fwd, bwd = calls[0], calls[1:]
    tag = "linear"
    x = view(xl.detach())
    wg, bg, rg = w.grad, b.grad if b is not None else None, res.grad if res is not None else None
    w, b = w.detach(), b.detach() if b is not None else None
    # ---- forward
    x2 = x.reshape(-1, K)
    same_bits(fwd.a, x2, "forward A is x")
    if form == "strided":
        assert fwd.a.data_ptr() == xl.data_ptr() and fwd.a.stride(0) == 197 * K, "strided x was copied"
    if form == "copy":
        assert fwd.a.is_contiguous() and fwd.a.data_ptr() != xl.data_ptr()
    assert same_ptr(fwd.b, w) and (b is None) == (fwd.bias is None) and (b is None or same_ptr(fwd.bias, b))
    assert not fwd.a_mn and not fwd.b_mn and fwd.act == ACTS[act]
    if res is not None:
        same_bits(fwd.residual, res, "forward residual")
    wants_z = act is not None and any(k in need for k in ("x", "w", "b"))
    assert (fwd.preact is not None) == wants_z, "pre-activation saved when no gradient reads it, or not saved"
    check_gemm(fwd, tag)
    same_bits(y.reshape(M, N), fwd.out, "y is the forward GEMM's output")
    # ---- backward: dz, then dgrad / wgrad / bias_grad in that order
    roles = [k for k in ("x", "w", "b") if k in need and (k != "b" or b is not None)]
    assert len(bwd) == len(roles), f"{len(bwd)} backward launches for {roles}"
    by = dict(zip(roles, bwd))
    dz = None
    if roles:
        dz = bwd[0].a                      # dgrad reads dz K-major, wgrad / bias_grad MN-major: the same [M, N]
        if act is None:
            same_bits(dz, dy, "dz is dy")
        else:
            from distributed_torch_horovod_gcp_b200.ops.gemm import act_backward
            same_bits(dz, act_backward(dy, fwd.preact, ACTS[act]), "dz = act_backward(dy, saved z)")
            ref, E = act_backward_bound(dy, fwd.preact, ACTS[act])
            _check(dz, ref, E, f"{tag} act_backward {act}")
        for r in bwd:
            same_bits(r.a, dz, f"{gemm_role(r)} reads dz")
    splits = None
    if "x" in by:
        r = by["x"]
        assert same_ptr(r.b, w) and r.b_mn and not r.a_mn and (r.M, r.N, r.K) == (M, K, N) and r.residual is None
        check_gemm(r, tag)
        same_bits(view(xl.grad), r.out.view(x.shape), "x.grad is dgrad's output")
        rest = xl.grad.clone()
        view(rest).zero_()
        assert float(rest.abs().max()) == 0.0, "gradient outside the view"
    if "w" in by:
        r = by["w"]
        same_bits(r.b, x2, "wgrad reads x as the forward did")
        assert r.b.data_ptr() == fwd.a.data_ptr(), "wgrad reads a copy of the saved x"
        assert r.a_mn and r.b_mn and (r.M, r.N, r.K) == (N, K, M)
        splits = r.splits
        assert splits == ops.gemm._splits_for(N, K, M)
        assert (r.out_mode, r.residual) == ((0, None) if splits == 1 else (2, None)), "store mode of a fresh dW"
        check_gemm(r, tag)
        same_bits(wg, r.out, "w.grad is wgrad's output")
    if "b" in by:
        r = by["b"]
        assert r.a_mn and r.b_mn and (r.M, r.N, r.K) == (N, 8, M) and r.out_mode == 1
        assert bool((r.b == 1).all()) and float(r.prev.abs().max()) == 0.0
        yb, Eb = check_gemm(r, tag)
        same_bits(bg, r.out[:, 0].to(bdt), "b.grad is acc[:, 0] in the bias dtype")
        _check(bg, yb[:, 0], bias_grad_bound(yb[:, 0], Eb[:, 0], bdt), f"{tag} bias_grad conversion")
    if "res" in need and res is not None:
        same_bits(rg, dy, "residual gradient is dy")
    # ---- end to end, float64 of the whole node on its exact inputs
    if roles:
        z64 = x2.double() @ w.double().t() + (b.double() if b is not None else 0)
        if act is None:
            dz64, Edz = dy.double(), torch.zeros(M, N, dtype=torch.float64, device="cuda")
        else:
            (_, _), (_, Ez) = epilogue_bounds(x2, w, 1.0, b, 0, None)     # the saved z against z*
            _, Eab = act_backward_bound(dy, fwd.preact, ACTS[act])
            if act == "relu":
                dz64 = dy.double() * (z64 > 0).double()
                Edz = dy.double().abs() * (z64.abs() <= Ez).double()
            else:
                dz64 = dy.double() * _gelu_grad64(z64)
                Edz = Eab + dy.double().abs() * GELU2_MAX * Ez
        if "x" in by:
            ref = dz64 @ w.double()
            _check(by["x"].out, ref, bf16_store(prop_gemm(Edz, dz, w.t(), N), ref), f"{tag} e2e dx")
        if "w" in by:
            ref = dz64.t() @ x2.double()
            _check(wg, ref, bf16_store(prop_gemm(Edz.t(), dz.t(), x2.t(), M), ref), f"{tag} e2e dW")
        if "b" in by:
            ref = dz64.sum(0)
            E = Edz.sum(0) + 2 * _pad64(M) * U32 * dz.double().abs().sum(0) + FLUSH
            _check(bg, ref, bias_grad_bound(ref, E, bdt), f"{tag} e2e db")
    return splits


# M, N, K, act, bias dtype, residual, x form, wgrad splits
LINEAR_CASES = [
    (1, 64, 128, "gelu", BF16, True, "2d", 1),
    (7, 72, 200, "relu", F32, False, "3d", 1),
    (127, 264, 72, None, None, True, "2d", 1),
    (129, 200, 264, "gelu", F32, True, "copy", 1),
    (127, 768, 768, "relu", None, False, "3d", 1),
    (394, 768, 768, "gelu", BF16, False, "strided", 1),
    (1000, 256, 256, "relu", BF16, True, "3d", 4),
    (1000, 768, 768, None, None, True, "strided", 4),
    (1000, 1000, 2048, None, F32, False, "2d", 1),          # the ResNet-50 head
    (129, 768, 3072, "gelu", BF16, False, "copy", 1),
    (7, 3072, 768, None, BF16, True, "2d", 1),
    (4096, 768, 768, "gelu", F32, True, "3d", 7),
    (4096, 3072, 768, "relu", BF16, False, "2d", 1),
]


def _case_id(c):
    M, N, K, act, bdt, res, form, s = c
    return f"M{M}-{N}x{K}-{act or 'none'}-{'nob' if bdt is None else str(bdt)[6:]}-{'res' if res else 'nores'}-{form}"


@gpu
@pytest.mark.parametrize("case", LINEAR_CASES, ids=_case_id)
def test_linear_stages(case, monkeypatch):
    M, N, K, act, bdt, with_res, form, splits = case
    ops = _ops()
    spy = Spy(monkeypatch, ops)
    need = {"x", "w"} | ({"b"} if bdt is not None else set()) | ({"res"} if with_res else set())
    got = run_linear(M, N, K, act, bdt, with_res, form, need, M + N + K, spy, ops)
    assert got == splits, f"wgrad took {got} splits, the case is meant for {splits}"


GRAD_SUBSETS = [frozenset(k for i, k in enumerate(("x", "w", "b", "res")) if m >> i & 1) for m in range(1, 16)]


@gpu
@pytest.mark.parametrize("need", GRAD_SUBSETS, ids=lambda s: "+".join(sorted(s)))
@pytest.mark.parametrize("act", [None, "relu", "gelu"], ids=["none", "relu", "gelu"])
def test_linear_every_grad_subset(act, need, monkeypatch):
    """Every non-empty subset of {x, weight, bias, residual} requiring grad.  With an activation, bias-only (bias-only
    fine-tuning) and residual-only need the saved pre-activation, or no activation gradient at all."""
    ops = _ops()
    spy = Spy(monkeypatch, ops)
    run_linear(129, 72, 136, act, BF16, True, "2d", need, 11, spy, ops)


# ================================================================================================ MLP
# M, D, Hd, bias dtype, residual
MLP_CASES = [
    (1, 64, 256, BF16, True),
    (7, 768, 3072, F32, False),
    (127, 64, 256, F32, True),
    (129, 768, 3072, BF16, True),
    (394, 768, 3072, BF16, True),
    (1000, 64, 256, BF16, False),
    (4096, 64, 256, F32, True),
    (4096, 768, 3072, BF16, True),
]


@gpu
@pytest.mark.parametrize("M,D,Hd,bdt,with_res", MLP_CASES,
                         ids=[f"M{c[0]}-{c[1]}-{c[2]}-{str(c[3])[6:]}-{'res' if c[4] else 'nores'}" for c in MLP_CASES])
def test_mlp_stages(M, D, Hd, bdt, with_res, monkeypatch):
    ops = _ops()
    spy = Spy(monkeypatch, ops)
    gen = torch.Generator(device="cuda").manual_seed(M + D)
    x = torch.randn(M, D, device="cuda", generator=gen).to(BF16).requires_grad_(True)
    w1 = (torch.randn(Hd, D, device="cuda", generator=gen) * 2.5 / math.sqrt(D)).to(BF16).requires_grad_(True)
    b1 = torch.randn(Hd, device="cuda", generator=gen).to(bdt).requires_grad_(True)
    w2 = (torch.randn(D, Hd, device="cuda", generator=gen) / math.sqrt(Hd)).to(BF16).requires_grad_(True)
    b2 = torch.randn(D, device="cuda", generator=gen).to(bdt).requires_grad_(True)
    res = torch.randn(M, D, device="cuda", generator=gen).to(BF16).requires_grad_(True) if with_res else None
    dy = torch.randn(M, D, device="cuda", generator=gen).to(BF16)
    y = ops.gemm.mlp(x, w1, b1, w2, b2, res)
    y.backward(dy)
    torch.cuda.synchronize()
    with torch.no_grad():
        _check_mlp(spy, ops, M, D, Hd, bdt, with_res, x, w1, b1, w2, b2, res, dy, y)


def _check_mlp(spy, ops, M, D, Hd, bdt, with_res, x, w1, b1, w2, b2, res, dy, y):
    calls = spy.of("gemm")
    assert [gemm_role(r) for r in calls] == ["fwd", "fwd", "dgrad act3", "wgrad", "bias_grad", "wgrad",
                                             "bias_grad", "dgrad"]
    fc1, fc2, dzc, dw2c, db2c, dw1c, db1c, dxc = calls
    tag = "mlp"
    for r in calls:
        check_gemm(r, tag)
    # hand-offs
    same_bits(fc1.a, x, "fc1 reads x")
    assert same_ptr(fc1.b, w1) and same_ptr(fc1.bias, b1) and fc1.act == 2 and fc1.preact is not None
    same_bits(fc2.a, fc1.out, "fc2 reads h")
    assert same_ptr(fc2.b, w2) and same_ptr(fc2.bias, b2) and fc2.act == 0
    if with_res:
        same_bits(fc2.residual, res, "fc2 residual")
    same_bits(y, fc2.out, "y is fc2's output")
    same_bits(dzc.a, dy, "fc2 dgrad reads dy")
    assert same_ptr(dzc.b, w2) and dzc.b_mn
    same_bits(dzc.residual, fc1.preact, "the fc2 dgrad's aux is the forward's saved z")
    same_bits(dw2c.a, dy, "dW2 reads dy")
    same_bits(dw2c.b, fc1.out, "dW2 reads h")
    same_bits(db2c.a, dy, "db2 reads dy")
    for r, what in ((dw1c, "dW1"), (db1c, "db1"), (dxc, "dx")):
        same_bits(r.a, dzc.out, f"{what} reads the act-3 output")
    same_bits(dw1c.b, x, "dW1 reads x")
    assert same_ptr(dxc.b, w1)
    for r, (n, k) in ((dw2c, (D, Hd)), (dw1c, (Hd, D))):
        assert r.splits == ops.gemm._splits_for(n, k, M) and r.out_mode == (0 if r.splits == 1 else 2)
    same_bits(x.grad, dxc.out, "x.grad")
    same_bits(w1.grad, dw1c.out, "w1.grad")
    same_bits(w2.grad, dw2c.out, "w2.grad")
    same_bits(b1.grad, db1c.out[:, 0].to(bdt), "b1.grad")
    same_bits(b2.grad, db2c.out[:, 0].to(bdt), "b2.grad")
    if with_res:
        same_bits(res.grad, dy, "residual gradient is dy")
    # end to end
    x, w1, b1, w2, b2 = (t.detach() for t in (x, w1, b1, w2, b2))
    x64, dy64 = x.double(), dy.double()
    z64 = x64 @ w1.double().t() + b1.double()
    (h64, Eh), (_, Ez) = epilogue_bounds(x, w1, 1.0, b1, 2, None)
    h = fc1.out
    ref = dy64.t() @ h64
    _check(dw2c.out, ref, bf16_store(prop_gemm(Eh.t(), h.t(), dy.t(), M).t(), ref), f"{tag} e2e dW2")
    ref = dy64.sum(0)
    E = 2 * _pad64(M) * U32 * dy64.abs().sum(0) + FLUSH
    _check(db2c.out[:, 0].to(bdt), ref, bias_grad_bound(ref, E, bdt), f"{tag} e2e db2")
    dh64 = dy64 @ w2.double()
    dz64 = dh64 * _gelu_grad64(z64)
    (_, Eact3), _ = epilogue_bounds(dy, w2.t(), 1.0, None, 3, fc1.preact)
    Edz = Eact3 + dh64.abs() * GELU2_MAX * Ez
    dz = dzc.out
    ref = dz64.t() @ x64
    _check(dw1c.out, ref, bf16_store(prop_gemm(Edz.t(), dz.t(), x.t(), M), ref), f"{tag} e2e dW1")
    ref = dz64.sum(0)
    E = Edz.sum(0) + 2 * _pad64(M) * U32 * dz.double().abs().sum(0) + FLUSH
    _check(db1c.out[:, 0].to(bdt), ref, bias_grad_bound(ref, E, bdt), f"{tag} e2e db1")
    ref = dz64 @ w1.double()
    _check(dxc.out, ref, bf16_store(prop_gemm(Edz, dz, w1.t(), Hd), ref), f"{tag} e2e dx")


# ================================================================================================ QKV
QKV_CASES = [(1, 192, BF16), (7, 768, F32), (127, 192, F32), (129, 768, BF16), (394, 768, BF16),
             (1000, 192, F32), (4096, 768, BF16), (4096, 192, F32)]


@gpu
@pytest.mark.parametrize("M,D,bdt", QKV_CASES, ids=[f"M{c[0]}-D{c[1]}-{str(c[2])[6:]}" for c in QKV_CASES])
def test_qkv_stages(M, D, bdt, monkeypatch):
    ops = _ops()
    spy = Spy(monkeypatch, ops)
    gen = torch.Generator(device="cuda").manual_seed(M * 3 + D)
    x = torch.randn(M, D, device="cuda", generator=gen).to(BF16).requires_grad_(True)
    w = (torch.randn(3 * D, D, device="cuda", generator=gen) / math.sqrt(D)).to(BF16).requires_grad_(True)
    b = torch.randn(3 * D, device="cuda", generator=gen).to(bdt).requires_grad_(True)
    gs = [torch.randn(M, D, device="cuda", generator=gen).to(BF16) * (i + 1) for i in range(3)]
    q, k, v = ops.gemm.qkv_proj(x.view(1, M, D), w, b)
    torch.autograd.backward([q, k, v], [g.view(1, M, D) for g in gs])
    torch.cuda.synchronize()
    with torch.no_grad():
        _check_qkv(spy, ops, M, D, bdt, x, w, b, gs, (q, k, v))


def _check_qkv(spy, ops, M, D, bdt, x, w, b, gs, outs):
    xg, wg, bg = x.grad, w.grad, b.grad
    x, w, b = x.detach(), w.detach(), b.detach()
    q, k, v = outs
    calls = spy.of("gemm")
    assert [gemm_role(r) for r in calls] == ["fwd"] * 3 + ["dgrad"] * 3 + ["wgrad"] * 3 + ["bias_grad"] * 3
    tag = "qkv"
    for r in calls:
        check_gemm(r, tag)
    ws = [w[i * D:(i + 1) * D] for i in range(3)]
    for i in range(3):
        f, dx_i, dw_i, db_i = calls[i], calls[3 + i], calls[6 + i], calls[9 + i]
        same_bits(f.a, x, "forward reads x")
        assert f.b.data_ptr() == ws[i].data_ptr() and f.b.shape == ws[i].shape, f"forward {i}: weight rows"
        assert f.bias.data_ptr() == b[i * D:].data_ptr()
        same_bits((q, k, v)[i].reshape(M, D), f.out, f"output {i}")
        same_bits(dx_i.a, gs[i], f"dgrad {i} reads its own output gradient")
        assert dx_i.b.data_ptr() == ws[i].data_ptr() and dx_i.b_mn
        if i == 0:
            assert dx_i.residual is None
        else:
            same_bits(dx_i.residual, calls[2 + i].out, f"dgrad {i} adds dgrad {i - 1}'s output")
        same_bits(dw_i.a, gs[i], f"wgrad {i} reads its output gradient")
        same_bits(dw_i.b, x, f"wgrad {i} reads x")
        assert dw_i.splits == ops.gemm._splits_for(D, D, M)
        same_bits(wg[i * D:(i + 1) * D], dw_i.out, f"rows {i * D}..{(i + 1) * D} of dW")
        same_bits(db_i.a, gs[i], f"bias_grad {i} reads its output gradient")
        same_bits(bg[i * D:(i + 1) * D], db_i.out[:, 0].to(bdt), f"db slice {i}")
    same_bits(xg, calls[5].out, "x.grad is the last dgrad's output")
    # end to end
    ref, E = qkv_dx_bound(gs, ws)
    _check(xg, ref, E, f"{tag} e2e dx (three bf16 roundings)")
    for i in range(3):
        ref = gs[i].double().t() @ x.double()
        E = 2 * _pad64(M) * U32 * (gs[i].double().abs().t() @ x.double().abs())
        _check(wg[i * D:(i + 1) * D], ref, bf16_store(E, ref), f"{tag} e2e dW")
        ref = gs[i].double().sum(0)
        E = 2 * _pad64(M) * U32 * gs[i].double().abs().sum(0) + FLUSH
        _check(bg[i * D:(i + 1) * D], ref, bias_grad_bound(ref, E, bdt), f"{tag} e2e db")


# ================================================================================================ bottleneck
def _block(kind, planes, seed):
    from distributed_torch_horovod_gcp_b200.models.resnet import Bottleneck
    torch.manual_seed(seed)
    if kind == "identity":
        cin, stride, ds = 4 * planes, 1, None
    else:
        cin, stride = (planes, 1) if kind == "proj_s1" else (2 * planes, 2)
        ds = nn.Sequential(nn.Conv2d(cin, 4 * planes, 1, stride, bias=False), nn.BatchNorm2d(4 * planes))
    blk = Bottleneck(cin, planes, stride, ds)
    with torch.no_grad():
        for m in blk.modules():
            if isinstance(m, nn.BatchNorm2d):
                m.weight.uniform_(0.5, 1.5)
                m.bias.uniform_(-0.2, 0.2)
    return blk.cuda().to(BF16).to(memory_format=torch.channels_last).train(), cin


def _freeze(blk, frozen):
    if frozen == "x" or frozen is None:
        return
    kind, name = frozen.split(":")
    mod = blk.downsample[0 if kind == "conv" else 1] if name == "ds" else getattr(blk, kind + name)
    for p in mod.parameters():
        p.requires_grad_(False)


def _nhwc(t):
    return t.to(BF16).contiguous(memory_format=torch.channels_last)


def _rows(t):
    N, C, H, W = t.shape
    return t.permute(0, 2, 3, 1).reshape(N * H * W, C)


# kind, planes, batch, map, what is frozen ("x", "conv:<unit>" or "bn:<unit>", unit 1 / 2 / 3 / ds)
BOTTLENECK_CASES = [
    ("identity", 16, 3, 7, None),
    ("identity", 64, 2, 14, "x"),
    ("identity", 16, 5, 2, "conv:2"),
    ("identity", 64, 3, 14, "conv:1"),
    ("proj_s1", 16, 3, 14, "bn:1"),
    ("proj_s1", 64, 3, 7, None),
    ("proj_s2", 16, 3, 14, None),
    ("proj_s2", 64, 2, 2, "conv:ds"),
    ("proj_s2", 16, 3, 2, "bn:3"),
]


@gpu
@pytest.mark.parametrize("kind,planes,batch,hw,frozen", BOTTLENECK_CASES,
                         ids=[f"{c[0]}-p{c[1]}-n{c[2]}-{c[3]}x{c[3]}-{c[4] or 'all'}" for c in BOTTLENECK_CASES])
def test_bottleneck_stages(kind, planes, batch, hw, frozen, monkeypatch):
    ops = _ops()
    blk, cin = _block(kind, planes, seed=planes + hw)
    _freeze(blk, frozen)
    gen = torch.Generator(device="cuda").manual_seed(batch * hw)
    x = _nhwc(torch.randn(batch, cin, hw, hw, device="cuda", generator=gen)).requires_grad_(frozen != "x")
    assert ops.bottleneck.supported(x, blk), "the block would take the per-op chain"
    spy = Spy(monkeypatch, ops)
    y = ops.bottleneck.bottleneck(x, blk)
    dy = _nhwc(torch.randn(y.shape, device="cuda", generator=gen))
    y.backward(dy)
    torch.cuda.synchronize()
    with torch.no_grad():
        _check_bottleneck(spy, ops, blk, x, y, dy)


def _check_bottleneck(spy, ops, blk, x, y, dy):
    check_launches(spy, "bottleneck")
    units = ops.bottleneck._units(blk)
    n = len(units)
    calls = spy.calls
    # ---- forward: (conv launch, bn_forward) per unit, in _units order
    fw = []
    for i, (conv, bn) in enumerate(units):
        c, f = calls[2 * i], calls[2 * i + 1]
        assert c.op in ("gemm", "conv_fprop") and f.op == "bn_forward" and f.bn is bn, (i, c.op, f.op)
        fw.append((c, f))
    inputs = {0: x.detach(), 1: fw[0][1].out_t, n - 1: fw[1][1].out_t}
    if n == 4:
        inputs[2] = x.detach()
    for i, (conv, bn) in enumerate(units):
        c, f = fw[i]
        xin = inputs[i]
        if c.op == "gemm":
            same_bits(c.a, _rows(xin), f"unit {i} GEMM reads its input")
            assert same_ptr(c.a, xin), f"unit {i}: the NHWC rows were copied"
            same_bits(c.b, conv.weight.detach().reshape(c.N, c.K), f"unit {i} weight")
            same_bits(_rows(f.x), c.out, f"bn {i} reads its conv's output")
        else:
            same_bits(c.x, xin, f"unit {i} conv reads its input")
            same_bits(f.x, c.out, f"bn {i} reads its conv's output")
        assert f.relu == (i != 2 or n == 3)
        assert (f.residual is None) == (i != n - 1)
    same_bits(fw[n - 1][1].residual, x.detach() if n == 3 else fw[2][1].out, "bn3's residual is the identity branch")
    same_bits(y.detach(), fw[n - 1][1].out, "the block's output is bn3's")
    # ---- backward, in the node's order: bn3, conv3; bn2, conv2; [downsample]; bn1, conv1
    bw = iter(calls[2 * n:])
    need_x = x.requires_grad

    def unit(i, dout, mask_owner, want_dx, residual=None, res_mask=None):
        conv, bn = units[i]
        c, f = fw[i]
        rb = next(bw)
        assert rb.op == "bn_backward" and rb.bn is bn, (i, rb.op)
        same_bits(rb.dy, dout, f"bn {i} backward reads its output gradient")
        assert same_ptr(rb.mask, fw[mask_owner][1].mask), f"bn {i} backward applies bn {mask_owner}'s sign bits"
        assert all(same_ptr(a, b) for a, b in zip(rb.ws, f.ws)), f"bn {i} backward reads its forward's statistics"
        if bn.weight.requires_grad:
            same_bits(bn.weight.grad, rb.dg, f"bn {i} .weight.grad")
            same_bits(bn.bias.grad, rb.db, f"bn {i} .bias.grad")
        else:
            assert bn.weight.grad is None and bn.bias.grad is None
        gemm_unit = c.op == "gemm"
        dx = None
        if want_dx:
            d = next(bw)
            if gemm_unit:
                assert d.op == "gemm" and gemm_role(d) == "dgrad", (i, d.op)
                same_bits(d.a, _rows(rb.out), f"unit {i} dgrad reads bn {i}'s dx")
                assert same_ptr(d.b, c.b) and d.b_mn
                if residual is None:
                    assert d.residual is None
                else:
                    same_bits(d.residual, _rows(residual), f"unit {i} dgrad residual")
                assert (d.res_mask is None) == (res_mask is None), f"unit {i} dgrad sign bits"
                if res_mask is not None:
                    assert same_ptr(d.res_mask, res_mask), f"unit {i} dgrad sign bits"
                N_, C_, H_, W_ = inputs[i].shape
                dx = d.out.view(N_, H_, W_, C_).permute(0, 3, 1, 2)
            else:
                assert d.op == "conv_dgrad", (i, d.op)
                same_bits(d.dy, rb.out, f"unit {i} dgrad reads bn {i}'s dx")
                assert same_ptr(d.w, c.w) and d.x_shape == tuple(inputs[i].shape)
                dx = d.out
        if conv.weight.requires_grad:
            wg = next(bw)
            if gemm_unit:
                assert wg.op == "gemm" and gemm_role(wg) == "wgrad", (i, wg.op)
                same_bits(wg.a, _rows(rb.out), f"unit {i} wgrad reads bn {i}'s dx")
                same_bits(wg.b, _rows(inputs[i]), f"unit {i} wgrad reads the activation its forward read")
                assert wg.splits == ops.gemm._splits_for(wg.M, wg.N, wg.K)
                same_bits(conv.weight.grad.reshape(wg.M, wg.N), wg.out, f"conv {i} .grad")
            else:
                assert wg.op == "conv_wgrad" and wg.returned, (i, wg.op)
                same_bits(wg.dy, rb.out, f"unit {i} wgrad reads bn {i}'s dx")
                same_bits(wg.x, inputs[i], f"unit {i} wgrad reads the activation its forward read")
                same_bits(conv.weight.grad, wg.out, f"conv {i} .grad")
        else:
            assert conv.weight.grad is None
        return dx

    d = unit(1, unit(n - 1, dy, n - 1, True), 1, True)
    if n == 4:
        # the downsample BN applies bn3's sign bits to dy; its dgrad is conv1's residual
        skip = unit(2, dy, n - 1, need_x)
        dx = unit(0, d, 0, need_x, skip, None)
    else:
        # identity: conv1's dgrad adds dy under bn3's sign bits
        dx = unit(0, d, 0, need_x, dy if need_x else None, fw[n - 1][1].mask if need_x else None)
    assert next(bw, None) is None, "unexpected launches after conv1's"
    if need_x:
        same_bits(x.grad, dx, "x.grad is conv1's dgrad output")
    else:
        assert x.grad is None


def _per_op(F2, blk, x):
    out = F2.conv_bn_act(x, blk.conv1, blk.bn1, relu=True)
    out = F2.conv_bn_act(out, blk.conv2, blk.bn2, relu=True)
    identity = x if blk.downsample is None else F2.conv_bn_act(x, blk.downsample[0], blk.downsample[1], relu=False)
    return F2.conv_bn_act(out, blk.conv3, blk.bn3, relu=True, residual=identity)


def _dgrad_of(spy, weight):
    """The data-gradient launch (GEMM or implicit-GEMM convolution) that read ``weight``, as an NCHW tensor."""
    rs = [r for r in spy.calls if (r.op == "gemm" and gemm_role(r) == "dgrad" and same_ptr(r.b, weight)) or
          (r.op == "conv_dgrad" and same_ptr(r.w, weight))]
    assert len(rs) == 1, len(rs)
    return rs[0]


@gpu
@pytest.mark.parametrize("kind,planes,batch,hw", [("identity", 16, 3, 7), ("proj_s1", 64, 3, 7),
                                                  ("proj_s2", 16, 3, 14), ("proj_s2", 64, 2, 2)])
def test_per_op_chain_stages(kind, planes, batch, hw, monkeypatch):
    """The same blocks through ``conv_bn_act`` (``_ConvFn`` on the 1x1 GEMM and the implicit-GEMM kernel,
    ``_BNActFn``): every launch against float64, bn3's dres is its masked dy, the downsample BN reads that dres, and
    x.grad is autograd's bf16 sum of conv1's dgrad and the skip gradient."""
    from distributed_torch_horovod_gcp_b200.ops import functional as F2
    ops = _ops()
    blk, cin = _block(kind, planes, seed=planes + hw + 1)
    gen = torch.Generator(device="cuda").manual_seed(batch * hw + 1)
    x = _nhwc(torch.randn(batch, cin, hw, hw, device="cuda", generator=gen)).requires_grad_(True)
    spy = Spy(monkeypatch, ops)
    y = _per_op(F2, blk, x)
    dy = _nhwc(torch.randn(y.shape, device="cuda", generator=gen))
    y.backward(dy)
    torch.cuda.synchronize()
    with torch.no_grad():
        check_launches(spy, "per-op")
        bwds = spy.of("bn_backward")
        (b3,) = [r for r in bwds if r.bn is blk.bn3]
        assert b3.write_dres and b3.dres is not None
        same_bits(b3.dy, dy, "bn3 backward reads dy")
        N_, C_, H_, W_ = x.shape

        def nchw(r):
            return r.out if r.op == "conv_dgrad" else r.out.view(N_, H_, W_, C_).permute(0, 3, 1, 2)

        g1 = nchw(_dgrad_of(spy, blk.conv1.weight))
        if blk.downsample is None:
            skip = b3.dres
        else:
            (bd,) = [r for r in bwds if r.bn is blk.downsample[1]]
            same_bits(bd.dy, b3.dres, "the downsample BN reads bn3's dres")
            assert bd.mask is None and not bd.write_dres
            skip = nchw(_dgrad_of(spy, blk.downsample[0].weight))
        ref = g1.double() + skip.double()
        _check(x.grad, ref, bf16_store(U32 * ref.abs(), ref), "per-op x.grad = bf16(dgrad + skip)")


@gpu
@pytest.mark.parametrize("relu", [True, False], ids=["relu", "norelu"])
def test_bnact_dres_paths(relu, monkeypatch):
    """``_BNActFn``'s residual gradient: with ReLU the masked dy its backward writes, without ReLU dy itself."""
    from distributed_torch_horovod_gcp_b200.ops import functional as F2
    ops = _ops()
    blk, cin = _block("identity", 16, seed=3)
    conv = nn.Conv2d(cin, 64, 1, bias=False).cuda().to(BF16).to(memory_format=torch.channels_last)
    gen = torch.Generator(device="cuda").manual_seed(5)
    x = _nhwc(torch.randn(3, cin, 7, 7, device="cuda", generator=gen))
    res = _nhwc(torch.randn(3, 64, 7, 7, device="cuda", generator=gen)).requires_grad_(True)
    spy = Spy(monkeypatch, ops)
    y = F2.conv_bn_act(x, conv, blk.bn3, relu=relu, residual=res)
    dy = _nhwc(torch.randn(y.shape, device="cuda", generator=gen))
    y.backward(dy)
    torch.cuda.synchronize()
    with torch.no_grad():
        check_launches(spy, "per-op")
        (rb,) = spy.of("bn_backward")
        assert rb.write_dres == relu
        if relu:
            same_bits(res.grad, rb.dres, "residual gradient is the BN backward's masked dy")
            assert torch.equal(_to2(rb.dres), bn_dz2(rb))
        else:
            same_bits(res.grad, dy, "residual gradient is dy")


# ================================================================================================ bucket slots
class _SinkNet(nn.Module):
    """A conv + BatchNorm (implicit-GEMM wgrad into its slot; γ / β straight into theirs on the first pass), a
    per-pixel linear whose wgrad takes split-K (256 x 64 over 2048 rows: 8 splits) and a head with one split."""

    def __init__(self):
        super().__init__()
        self.conv = nn.Conv2d(16, 64, 3, 1, 1, bias=False)
        self.bn = nn.BatchNorm2d(64)
        self.fc1 = nn.Linear(64, 256)
        self.fc2 = nn.Linear(256, 16)

    def forward(self, x, gemm, F2):
        h = F2.conv_bn_act(x, self.conv, self.bn, relu=True)
        B, C, H, W = h.shape
        u = gemm.linear(_rows(h), self.fc1.weight, self.fc1.bias, act="relu")
        return gemm.linear(u.view(B, H * W, -1).mean(1), self.fc2.weight, self.fc2.bias)


SLOTS = ("conv.weight", "bn.weight", "bn.bias", "fc1.weight", "fc2.weight")


def _run_sink_passes(hvd, ops, check):
    """Two backward passes of ``backward_passes_per_step=3`` recorded by spies, handed with the gradients after each
    to ``check`` before the third pass launches the buckets and the optimizer moves the weights."""
    from distributed_torch_horovod_gcp_b200.ops import functional as F2
    torch.manual_seed(0)
    model = _SinkNet().cuda().to(BF16).to(memory_format=torch.channels_last)
    with torch.no_grad():
        model.bn.weight.uniform_(0.5, 1.5)
        model.bn.bias.uniform_(-0.2, 0.2)
    opt = hvd.DistributedOptimizer(torch.optim.SGD(model.parameters(), lr=0.05, momentum=0.9),
                                   named_parameters=model.named_parameters(), backward_passes_per_step=3)
    assert opt.fused_engine is not None
    gen = torch.Generator(device="cuda").manual_seed(2)
    x = _nhwc(torch.randn(8, 16, 16, 16, device="cuda", generator=gen))
    g = torch.randn(8, 16, device="cuda", generator=gen).to(BF16)
    passes = []
    try:
        for _ in range(2):
            mp = pytest.MonkeyPatch()
            try:
                spy = Spy(mp, ops)
                model(x, ops.gemm, F2).backward(g)
                torch.cuda.synchronize()
            finally:
                mp.undo()
            passes.append((spy, {n: p.grad.detach().clone() for n, p in model.named_parameters()}))
        with torch.no_grad():
            check(model, passes)
        model(x, ops.gemm, F2).backward(g)
        opt.step()
        opt.zero_grad()
        torch.cuda.synchronize()
    finally:
        opt.remove_hooks()


def _stage_values(spy):
    """Per slot: (the stage's output, float64 dW of its recorded inputs and its bound as one bf16 value, in the
    parameter's shape, and the launch record)."""
    out = {}
    M = 8 * 16 * 16
    for name, (N, K, rows) in (("fc1.weight", (256, 64, M)), ("fc2.weight", (16, 256, 8))):
        (r,) = [r for r in spy.of("gemm") if gemm_role(r) == "wgrad" and (r.M, r.N, r.K) == (N, K, rows)]
        A, B = gemm_operands(r)
        ref = A.double() @ B.double().t()
        E1 = bf16_store(2 * _pad64(rows) * U32 * (A.double().abs() @ B.double().abs().t()), ref)
        out[name] = (r.out, ref, E1, r)
    (c,) = spy.of("conv_wgrad")
    ref, mag = _wgrad_ref(c.x, c.dy, 3, c.stride, c.pad)
    E1 = bf16_store(2 * _pad64(M) * U32 * mag, ref)
    out["conv.weight"] = (c.out, ref.permute(0, 3, 1, 2), E1.permute(0, 3, 1, 2), c)
    (rb,) = spy.of("bn_backward")
    f = bn_forward_of(spy, rb)
    N, C, H, W = rb.x.shape
    _, (dgr, dgb), (dbr, dbb) = bn_bwd_bounds(_to2(rb.x), bn_dz2(rb), f.gamma, f.D,
                                              standalone_depth(N * H * W, C, _sms()), True)
    out["bn.weight"] = (rb.dg, dgr, dgb, rb)
    out["bn.bias"] = (rb.db, dbr, dbb, rb)
    return out


@gpu
def test_bucket_slot_accumulation(monkeypatch):
    """``backward_passes_per_step=3`` through the fused engine: after pass 1 every slot holds its stage's output bit
    for bit; after pass 2 it lies within ``accumulate_bound`` of fl(prev + dW*), elementwise, both where the kernels
    write the slots (split-K ``out_mode=1``, the aliased ``residual=dw``, the conv wgrad's add; γ / β fall back to
    autograd) and where autograd's AccumulateGrad does (``grad_sink._ENABLED = False``)."""
    monkeypatch.setenv("B200DP_FUSED_SINGLE", "1")
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK", "LOCAL_WORLD_SIZE", "HOROVOD_TIMELINE"):
        monkeypatch.delenv(k, raising=False)
    import distributed_torch_horovod_gcp_b200.torch as hvd
    ops = _ops()
    hvd.shutdown()
    hvd.init()
    try:
        for enabled in (True, False):
            ops.grad_sink._ENABLED = enabled
            _run_sink_passes(hvd, ops, lambda model, passes: _check_slots(enabled, model, passes))
    finally:
        ops.grad_sink._ENABLED = True
        hvd.shutdown()


def _check_slots(enabled, model, passes):
    (spy1, g1), (spy2, g2) = passes
    tag = f"bucket {'sink' if enabled else 'autograd'}"
    check_launches(spy1, tag + " pass 1")
    check_launches(spy2, tag + " pass 2")
    s1, s2 = _stage_values(spy1), _stage_values(spy2)
    for name in SLOTS:
        shape = g1[name].shape
        assert torch.equal(g1[name], s1[name][0].view(shape)), f"{tag} {name}: slot after pass 1"
        _, ref2, E2, _ = s2[name]
        ref2, E2 = ref2.reshape(shape), E2.reshape(shape)
        _check(g2[name], g1[name].double() + ref2, accumulate_bound(g1[name], ref2, E2),
               f"{tag} pass 2 slot")
    fc1, fc2 = s1["fc1.weight"][3], s1["fc2.weight"][3]
    assert fc1.splits == 8 and fc2.splits == 1, (fc1.splits, fc2.splits)
    a1, a2 = s2["fc1.weight"][3], s2["fc2.weight"][3]
    c1, c2 = s1["conv.weight"][3], s2["conv.weight"][3]
    b1, b2 = s1["bn.weight"][3], s2["bn.weight"][3]
    if enabled:
        p = dict(model.named_parameters())
        assert fc1.out_mode == 2 and a1.out_mode == 1, "split-K: store on pass 1, add on pass 2"
        assert fc2.residual is None and fc2.out_mode == 0 and a2.alias, "one split: residual=dw on pass 2"
        same_bits(a1.prev, g1["fc1.weight"], "the split-K add starts from the slot")
        same_bits(a2.residual, g1["fc2.weight"], "residual=dw reads the slot")
        assert a1.out_ptr == p["fc1.weight"].grad.data_ptr() == fc1.out_ptr
        assert a2.out_ptr == p["fc2.weight"].grad.data_ptr() == fc2.out_ptr
        assert c1.sink and c1.prev is None and c2.sink and c2.prev is not None
        same_bits(c2.prev, g1["conv.weight"], "the conv wgrad adds onto the slot")
        assert b1.direct and not b2.direct, "γ / β: straight into the slots on pass 1 only"
    else:
        for r in (a1, a2):
            assert r.out_mode != 1 and not r.alias
        assert not (c1.sink or c2.sink or b1.direct or b2.direct)


# ================================================================================================ the bounds themselves (CPU)
def test_declared_split_counts():
    """The split counts the GEMM cases above are meant to exercise (no device needed: ``_splits_for`` is host code)."""
    from distributed_torch_horovod_gcp_b200.ops.gemm import _splits_for
    for M, N, K, *_, s in LINEAR_CASES:
        assert _splits_for(N, K, M) == s, (M, N, K)
    assert {_splits_for(N, K, M) for M, N, K, *_ in LINEAR_CASES} >= {1, 4, 7}
    assert _splits_for(256, 64, 2048) == 8 and _splits_for(16, 256, 8) == 1       # _SinkNet
    assert _splits_for(256, 64, 4096) == 16 and _splits_for(192, 192, 4096) == 16  # MLP 64/256, QKV 192


def _bf(t):
    return t.to(BF16)


def _cpu_gelu_case(n=4096, seed=0):
    g = torch.Generator().manual_seed(seed)
    z = _bf(torch.linspace(-9, 9, n) + 0.01 * torch.randn(n, generator=g))
    dy = _bf(torch.randn(n, generator=g) * 4)
    return dy, z


def _emulated(name):
    """(out, float64 reference, bound) of one composed step, emulated in fp32 on the CPU."""
    from distributed_torch_horovod_gcp_b200.ops.gemm import act_backward
    g = torch.Generator().manual_seed(1)
    if name == "act_backward gelu":
        dy, z = _cpu_gelu_case()
        ref, E = act_backward_bound(dy, z, 2)
        return act_backward(dy, z, 2), ref, E
    if name == "act_backward relu":
        dy, z = _cpu_gelu_case()
        ref, E = act_backward_bound(dy, z, 1)
        return act_backward(dy, z, 1), ref, E
    if name == "bias_grad conversion":
        dz = _bf(torch.randn(1000, 64, generator=g))
        acc = dz.float().sum(0)                                    # some fp32 order
        ref = dz.double().sum(0)
        E = 2 * _pad64(1000) * U32 * dz.double().abs().sum(0) + FLUSH
        return acc.to(BF16), ref, bias_grad_bound(ref, E, BF16)
    if name == "accumulate step":
        prev = _bf(torch.randn(4096, generator=g))
        d32 = torch.randn(4096, generator=g) * torch.logspace(-3, 1, 4096)
        ref = d32.double()
        E1 = bf16_store(torch.zeros_like(ref), ref)
        out_autograd = _bf(prev.float() + _bf(d32).float())
        return out_autograd, prev.double() + ref, accumulate_bound(prev, ref, E1)
    if name == "accumulate step (kernel)":
        prev = _bf(torch.randn(4096, generator=g))
        d32 = torch.randn(4096, generator=g) * torch.logspace(-3, 1, 4096)
        ref = d32.double()
        E1 = bf16_store(torch.zeros_like(ref), ref)
        return _bf(prev.float() + d32), prev.double() + ref, accumulate_bound(prev, ref, E1)
    if name == "qkv dx chain":
        M, D = 64, 192
        gs = [_bf(torch.randn(M, D, generator=g)) for _ in range(3)]
        ws = [_bf(torch.randn(D, D, generator=g) / math.sqrt(D)) for _ in range(3)]
        dx = None
        for gi, wi in zip(gs, ws):
            acc = gi.float() @ wi.float()
            dx = _bf(acc if dx is None else acc + dx.float())
        ref, E = qkv_dx_bound(gs, ws)
        return dx, ref, E
    raise KeyError(name)


CPU_STEPS = ["act_backward gelu", "act_backward relu", "bias_grad conversion", "accumulate step",
             "accumulate step (kernel)", "qkv dx chain"]


@pytest.mark.parametrize("name", CPU_STEPS)
def test_cpu_emulation_within_bounds(name):
    out, ref, E = _emulated(name)
    _check(out, ref, E, f"cpu {name}")


@pytest.mark.parametrize("name", [n for n in CPU_STEPS if n != "act_backward relu"])
def test_cpu_tightest_element_beyond_bound_fails(name):
    """The element closest to its bound, moved to 1.01x the bound (in float64), fails; at 0.99x it passes."""
    out, ref, E = _emulated(name)
    err = (out.double() - ref).abs()
    ratio = torch.where(E > 0, err / E.clamp_min(1e-300), torch.zeros_like(err))
    i = int(torch.argmax(ratio))
    assert 0 < float(ratio.reshape(-1)[i]) <= 1
    for f, ok in ((1.01, False), (0.99, True)):
        moved = out.double().clone().reshape(-1)
        s = 1.0 if float((out.double() - ref).reshape(-1)[i]) >= 0 else -1.0
        moved[i] = ref.reshape(-1)[i] + s * f * E.reshape(-1)[i]
        try:
            _check(moved.view(ref.shape), ref, E, "cpu tightness probe")
            passed = True
        except AssertionError:
            passed = False
        assert passed == ok, (f, ok)
    fp64_bounds._WORST.pop("cpu tightness probe", None)


def test_cpu_relu_act_backward_is_exact():
    dy, z = _cpu_gelu_case()
    from distributed_torch_horovod_gcp_b200.ops.gemm import act_backward
    assert torch.equal(act_backward(dy, z, 1), torch.where(z > 0, dy, torch.zeros_like(dy)))
