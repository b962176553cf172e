"""ResNet-50 kernel numerics against float64: the GEMM epilogues (csrc/sm90_common.cuh ``epilogue_frag``), the
implicit-GEMM convolution forward and data gradient (csrc/conv_sm90.cu), the BatchNorm forward / backward /
inference kernels, max / average pooling and the stem im2col (csrc/elementwise.cu), element by element.

Every reference is the operation in float64 on the exact bf16 (or fp32) values the kernel saw.  Every bound is
derived from the roundings the kernel performs (each ``*_bounds`` helper writes its derivation out), not fitted to
observed errors.  u = 2^-24 is the fp32 unit roundoff, U_BF16 = 2^-8 the relative error of a bf16 store.  A sum of
n fp32 terms in any order is within 2 n u sum|terms| of the exact sum (the factor 2 covers the tensor cores'
internal accumulation); a sum whose order is known is within 1.01 D u sum|terms|, D the longest chain of
additions any term goes through.  Zero-padded reduction chunks (TMA out-of-bounds fill) add exact zeros, but
they are counted as terms.

What is not bounded here because ``test_gpu_reductions.py`` already does: split-K order, the BatchNorm
statistics sums themselves and the conv weight gradient.  Here the outputs computed FROM those sums are checked.

Where the one-pass variance (E[x^2] - mean^2 in fp32) stands: at |mean|/std = 8 and M = 8*56*56 the kernel's
BatchNorm output is compared with ``nn.BatchNorm2d`` in bf16 on the same input and must be within twice its
error (``test_bn_one_pass_variance_vs_library``); the bound of every BN test keeps the cancellation term
(2 |mean| E_mean + E_sumsq) explicit, so at |mean|/std = 64 it is the bound, not a comparison, that holds.
"""
import math

import pytest
import torch
import torch.nn.functional as F

import fp64_bounds
from fp64_bounds import U32, U_BF16, assert_within_bound, report_ratios

gpu = pytest.mark.gpu

# Accuracy of the approximate fp32 instructions, as documented (PTX ISA, CUDA C Programming Guide), with a factor
# of 2 to spare: rsqrtf (2 ulp), __fdividef (2 ulp), ex2.approx (2 ulp).
U_RSQRT = 2.0 ** -21
U_DIV = 2.0 ** -21
U_EX2 = 2.0 ** -21
FLUSH = 2.0 ** -126       # a subnormal flushed to zero (add.ftz)
AS_ERF = 1.5e-7           # Abramowitz-Stegun 7.1.26: |erf_AS(x) - erf(x)| <= 1.5e-7 in exact arithmetic
AS_COEF = [0.254829592, -0.284496736, 1.421413741, -1.453152027, 1.061405429]


@pytest.fixture(scope="module", autouse=True)
def _report_ratios():
    yield
    report_ratios()


def _cdiv(a, b):
    return -(-a // b)


def _pad64(n):
    return 64 * _cdiv(n, 64)


def bf16_store(E, ref):
    """Bound after rounding a value that is within E of ref to bf16: |bf16(v) - v| <= U_BF16 |v|."""
    return (1 + U_BF16) * E + U_BF16 * ref.abs()


def _check(out, ref, bound, group):
    assert_within_bound(out, ref, group=group, terms=[(1.0, bound)])


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _nhwc(t):
    return t.to(torch.bfloat16).contiguous(memory_format=torch.channels_last)


def _nan_nhwc(*shape):
    """A bf16 channels_last output buffer filled with NaN: an element the kernel does not write shows."""
    return torch.empty(shape, device="cuda", dtype=torch.bfloat16, memory_format=torch.channels_last).fill_(float("nan"))


# ================================================================================================ GEMM epilogue
def _erf_poly_constants():
    """Two properties of the A&S polynomial P(t) = sum a_i t^i on t = 1/(1 + 0.3275911 |x|) in (0, 1], evaluated
    in float64 on a grid of 10^6 points (+1 % for the grid):
    K_t = max |d log(t P(t)) / d log t| (how a relative error of t grows in q = t P(t) e^(-x^2)), and
    H = max sum |a_i| t^i / P(t) (the amplification of the Horner roundings and the fp32 coefficients)."""
    t = torch.linspace(1e-9, 1.0, 1_000_001, dtype=torch.float64)
    P = sum(c * t ** i for i, c in enumerate(AS_COEF))
    dP = sum(i * c * t ** (i - 1) for i, c in enumerate(AS_COEF) if i)
    assert float(P.min()) > 0
    K_t = float((1 + t * dP / P).abs().max()) * 1.01
    H = float((sum(abs(c) * t ** i for i, c in enumerate(AS_COEF)) / P).max()) * 1.01
    return K_t, H


_KT, _H = _erf_poly_constants()


def fast_erf_err(x):
    """Bound on |fast_erf(x) - erf(x)| (float64 tensor x), derived from sm90_common.cuh ``fast_erf``:
    y = 1 - q with q = P(t) t e^(-x^2), and
    - t = __fdividef(1, fma(c, |x|, 1)): the fma, the fp32 constant c and the division, 2u + U_DIV relative,
      which moves q by K_t times that;
    - Horner (4 fma) with fp32 coefficients: (4 + 1)u H relative, doubled for safety;
    - poly * t * e: 2u;  e = __expf(-(|x| |x|)): the rounded square and the rounded x log2(e) inside __expf
      move the exponent by 2u x^2 (relative 2.02 u x^2 of e), ex2.approx adds U_EX2;
    - 1 - q: u (|y| <= 1).
    q itself is at most erfc(|x|) + AS_ERF.  Together with the A&S error: AS_ERF + q (rho_0 + 2.02 u x^2) + u."""
    rho0 = 1.01 * (_KT * (2 * U32 + U_DIV) + 10 * U32 * _H + 2 * U32 + U_EX2)
    q = torch.erfc(x.abs()) + AS_ERF
    return AS_ERF + q * (rho0 + 2.02 * U32 * x * x) + U32


def _gelu64(z):
    return 0.5 * z * (1 + torch.erf(z / math.sqrt(2.0)))


def _gelu_grad64(a):
    return 0.5 * (1 + torch.erf(a / math.sqrt(2.0))) + a * torch.exp(-0.5 * a * a) / math.sqrt(2 * math.pi)


def epilogue_bounds(A, B, alpha=1.0, bias=None, act=0, residual=None, out_fp32=False):
    """float64 references and bounds of ``epilogue_frag``'s outputs for C = A B^T (A [M, K], B [N, K], exact values).

    1. acc: fp32 accumulation of 64 ceil(K / 64) products (the K tail is zero-filled): E = 2 n u (|A||B|^T).
    2. v = fl(alpha acc) if alpha != 1, then fl(v + bias) (bf16 or fp32 bias): each rounding adds u (|z*| + E),
       z* = alpha A B^T + bias.  ``preact`` = bf16(v): bf16_store(E, z*) (one bf16 rounding of the fp32 value).
    3. act 1: ReLU (1-Lipschitz, E unchanged).  act 2: gelu_erf(v) = fl(fl(0.5 v) fl(1 + fast_erf(fl(v c)))):
       |gelu'| <= 1.13 carries E; fast_erf_err at v (taken at |z*| - E), its argument rounded twice (2.02 u |v c|,
       |erf'| <= 2/sqrt(pi)), and 2 roundings of the product: 0.5 |v| (E_erf + 2.02 u (|1 + erf| + E_erf)).
       act 3: v gelu_erf_grad(aux), aux the bf16 residual read exactly: cdf = 0.5 (1 + fast_erf) within
       0.5 E_erf + u, pdf = fl(0.39894f __expf(fl(-0.5 a) a)) within (3.03 u + U_EX2 + 1.01 u a^2) pdf, the
       x pdf product and the sum 2u; then the product v g (E |g| + |z| E_g + u).  act 4: v where aux > 0, else 0.
    4. residual (act 0-2): fl(v + r), u (|y*| + E).
    5. the store: bf16 (bf16_store) or fp32 through add.ftz (+ FLUSH)."""
    a64, b64 = A.double(), B.double()
    K = A.shape[1]
    p = a64 @ b64.t()
    E = 2 * _pad64(K) * U32 * (a64.abs() @ b64.abs().t())
    z = p
    if alpha != 1.0:
        z = alpha * p
        E = abs(alpha) * E
        E = E + U32 * (z.abs() + E)
    if bias is not None:
        z = z + bias.double()
        E = E + U32 * (z.abs() + E)
    pre = (z, bf16_store(E, z))
    y = z
    if act == 1:
        y = z.clamp_min(0)
    elif act == 2:
        c = 1 / math.sqrt(2.0)
        zlo = (z.abs() - E).clamp_min(0)
        Ee = fast_erf_err(zlo * c) + 2.02 * U32 * (z.abs() + E) * c * (2 / math.sqrt(math.pi))
        y = _gelu64(z)
        E = 1.13 * E + 0.5 * (z.abs() + E) * (Ee + 2.02 * U32 * ((1 + torch.erf(z * c)).abs() + Ee))
    elif act in (3, 4):
        a = residual.double()
        if act == 3:
            g = _gelu_grad64(a)
            pdf = torch.exp(-0.5 * a * a) / math.sqrt(2 * math.pi)
            Eg = 0.5 * fast_erf_err(a / math.sqrt(2.0)) + 0.5 * 2.02 * U32 * (a.abs() / math.sqrt(2.0)) \
                * (2 / math.sqrt(math.pi)) + U32 + a.abs() * pdf * (3.03 * U32 + U_EX2 + 1.01 * U32 * a * a) \
                + 2.02 * U32 * (g.abs() + a.abs() * pdf)
            y = z * g
            E = E * (g.abs() + Eg) + z.abs() * Eg
            E = E + U32 * (y.abs() + E)
        else:
            keep = (a > 0).double()
            y, E = z * keep, E * keep
    if residual is not None and act <= 2:
        y = y + residual.double()
        E = E + U32 * (y.abs() + E)
    out = (y, E + FLUSH) if out_fp32 else (y, bf16_store(E, y))
    return out, pre


def _gemm_mod():
    from distributed_torch_horovod_gcp_b200.ops import gemm, kernels
    assert kernels.has("gemm"), "libb200dp_kernels.so not loaded / gemm symbol missing"
    return gemm


# path: (alpha, bias dtype, act, residual kind, preact, out_mode, out dtype, res_mask)
GEMM_PATHS = {
    "plain": (1.0, None, 0, None, False, 0, torch.bfloat16, False),
    "res_only": (1.0, None, 0, "plain", False, 0, torch.bfloat16, False),
    "res_only_cancel": (1.0, None, 0, "cancel", False, 0, torch.bfloat16, False),
    "res_mask": (1.0, None, 0, "plain", False, 0, torch.bfloat16, True),
    "bias_bf16_preact": (1.0, torch.bfloat16, 0, None, True, 0, torch.bfloat16, False),
    "bias_f32_alpha_relu_res": (-1.5, torch.float32, 1, "plain", True, 0, torch.bfloat16, False),
    "bias_cancel": (0.75, torch.float32, 0, "cancel", True, 0, torch.bfloat16, False),
    "gelu_res": (0.75, torch.bfloat16, 2, "plain", True, 0, torch.bfloat16, False),
    "act3_gelu_grad": (1.0, None, 3, "aux", False, 0, torch.bfloat16, False),
    "act4_relu_grad": (1.0, None, 4, "aux", False, 0, torch.bfloat16, False),
    "store_bf16": (1.25, torch.float32, 2, None, True, 2, torch.bfloat16, False),
    "store_fp32": (-0.5, None, 0, None, False, 2, torch.float32, False),
}
# M tails 1 / 127 / 129 / 1000, N tails 8 / 72 / 200 / 264, K tails 8 / 72 / 200; extra = ldc - N
GEMM_SHAPES = [(1, 8, 8, 8), (127, 72, 72, 0), (129, 200, 200, 24), (1000, 264, 72, 8), (1000, 8, 200, 0),
               (129, 264, 8, 16)]
GEMM_MASK_SHAPES = [(1, 64, 8, 0), (127, 192, 72, 0), (1000, 320, 200, 0), (129, 64, 200, 0)]
BLOCK_NS = (0, 64, 128, 256)


def gemm_inputs(M, N, K, path, seed):
    """Operands of one path.  GELU paths put the pre-activation over about +-8 (the erf tails); act 3 / 4 read an
    aux uniform on (-6, 6); the cancellation paths take residual = -bf16(alpha A B^T + bias), so the exact result
    is the (small) rounding residue and a product rounded before the add would be off by U_BF16 |A B^T|."""
    alpha, bdt, act, rk, _, _, _, _ = GEMM_PATHS[path]
    g = torch.Generator().manual_seed(seed)
    A = torch.randn(M, K, generator=g).bfloat16()
    scale = 2.5 if act == 2 else 1.0
    B = (torch.randn(N, K, generator=g) * scale / math.sqrt(K)).bfloat16()
    bias = None
    if bdt is not None:
        bias = (torch.rand(N, generator=g) * 6 - 3 if act == 2 else torch.randn(N, generator=g)).to(bdt)
    res = None
    if rk == "plain":
        res = torch.randn(M, N, generator=g).bfloat16()
    elif rk == "aux":
        res = (torch.rand(M, N, generator=g) * 12 - 6).bfloat16()
    elif rk == "cancel":
        z = alpha * (A.double() @ B.double().t())
        if bias is not None:
            z = z + bias.double()
        res = (-z).bfloat16()
    return A, B, bias, res


def run_gemm_path(path, M, N, K, extra, block_n, seed):
    alpha, bdt, act, rk, want_pre, out_mode, odt, use_mask = GEMM_PATHS[path]
    gm = _gemm_mod()
    A, B, bias, res = gemm_inputs(M, N, K, path, seed)
    ldc = N + extra
    dev = "cuda"
    b_mn = rk is not None            # the residual / aux paths are dgrad GEMMs: B is MN-major
    a = A.to(dev)
    b = B.t().contiguous().to(dev) if b_mn else B.to(dev)
    out_big = torch.full((M, ldc), float("nan"), dtype=odt, device=dev)
    res_big = pre_big = bits = None
    res_used = res
    if res is not None:
        res_big = torch.full((M, ldc), float("nan"), dtype=torch.bfloat16, device=dev)
        res_big[:, :N] = res.to(dev)
    if use_mask:
        gk = torch.Generator().manual_seed(seed + 1)
        keep = torch.rand(M, N, generator=gk) > 0.4
        bits = (keep.view(M, N // 8, 8).to(torch.uint8) << torch.arange(8, dtype=torch.uint8)).sum(2).to(torch.uint8)
        res_used = res * keep.bfloat16()
        bits = bits.contiguous().to(dev)
    if want_pre:
        pre_big = torch.full((M, ldc), float("nan"), dtype=torch.bfloat16, device=dev)
    gm.gemm(a, b, out_big[:, :N], M, N, K, b_mn=b_mn, bias=bias.to(dev) if bias is not None else None,
            residual=res_big[:, :N] if res_big is not None else None,
            preact=pre_big[:, :N] if pre_big is not None else None, act=act, out_mode=out_mode, alpha=alpha,
            block_n=block_n, res_mask=bits)
    torch.cuda.synchronize()
    (y, yb), (z, zb) = epilogue_bounds(A.to(dev), B.to(dev), alpha, bias.to(dev) if bias is not None else None,
                                       act, res_used.to(dev) if res_used is not None else None,
                                       out_fp32=odt == torch.float32)
    tag = "fp32" if odt == torch.float32 else "bf16"
    _check(out_big[:, :N], y, yb, f"gemm epilogue {path}")
    if want_pre:
        _check(pre_big[:, :N], z, zb, "gemm epilogue preact")
        assert bool(pre_big[:, N:].isnan().all()), "preact written past column N"
    if extra:
        assert bool(out_big[:, N:].isnan().all()), f"{tag} output written past column N"
    return out_big[:, :N]


@gpu
@pytest.mark.parametrize("shape", GEMM_SHAPES, ids=lambda s: "x".join(map(str, s)))
@pytest.mark.parametrize("path", [p for p in GEMM_PATHS if p != "res_mask"])
def test_gemm_epilogue_vs_fp64(path, shape):
    M, N, K, extra = shape
    outs = [run_gemm_path(path, M, N, K, extra, bn, seed=M + N + K) for bn in BLOCK_NS]
    for o in outs[1:]:      # the tile width changes which thread rounds what, never the value
        assert torch.equal(o.view(torch.int16 if o.dtype == torch.bfloat16 else torch.int32),
                           outs[0].view(torch.int16 if o.dtype == torch.bfloat16 else torch.int32))


@gpu
@pytest.mark.parametrize("shape", GEMM_MASK_SHAPES, ids=lambda s: "x".join(map(str, s)))
def test_gemm_epilogue_res_mask_vs_fp64(shape):
    M, N, K, extra = shape
    for bn in BLOCK_NS:
        run_gemm_path("res_mask", M, N, K, extra, bn, seed=M + N)


@gpu
def test_gemm_cancellation_regime_is_not_vacuous():
    """The cancellation paths leave results of about U_BF16 |A B^T|: a product rounded to bf16 before the add
    would be off by as much as the result itself, far outside the bound.  Check the inputs do that."""
    A, B, bias, res = gemm_inputs(1000, 264, 72, "res_only_cancel", seed=1)
    p = A.double() @ B.double().t()
    y = p + res.double()
    assert float(y.abs().max()) <= 2 * U_BF16 * float(p.abs().max())
    assert float((p.bfloat16().double() + res.double()).abs().max()) == 0.0


# ================================================================================================ convolution
def conv_fprop_ref(x, w, stride, pad):
    x64, w64 = x.double(), w.double()
    return F.conv2d(x64, w64, None, stride, pad), F.conv2d(x64.abs(), w64.abs(), None, stride, pad)


def conv_dgrad_ref(dy, w, x_shape, stride, pad):
    g = torch.nn.grad.conv2d_input
    return (g(x_shape, w.double(), dy.double(), stride, pad),
            g(x_shape, w.double().abs(), dy.double().abs(), stride, pad))


def conv_bound(ref, mag, n_red):
    """fp32 accumulation of n_red = taps x 64-channel chunks x 64 products, then one bf16 store."""
    return bf16_store(2 * n_red * U32 * mag, ref)


def _border(t):
    """[N, C, H, W] mask of the first / last row and column: where the TMA out-of-bounds fill supplies taps."""
    H, W = t.shape[2], t.shape[3]
    m = torch.zeros(H, W, dtype=torch.bool, device=t.device)
    m[0] = m[-1] = True
    m[:, 0] = m[:, -1] = True
    return m.expand_as(t)


def _check_split(out, ref, bound, group):
    bm = _border(ref)
    for sel, name in ((bm, "border"), (~bm, "interior")):
        if bool(sel.any()):
            _check(out[sel], ref[sel], bound[sel], f"{group} {name}")


CONV_CASES = [
    # N, Cin, H, W, Cout, R, stride
    (3, 16, 7, 7, 72, 3, 1),       # odd batch, 7x7, Cin 16 (reduction tail inside one 64-channel chunk)
    (3, 24, 14, 14, 200, 3, 1),
    (2, 40, 14, 14, 72, 3, 2),
    (5, 24, 2, 2, 72, 3, 2),       # 2x2 map, stride 2: one output pixel
    (3, 40, 2, 2, 200, 1, 2),
    (2, 16, 12, 20, 72, 1, 2),     # W != H
    (1, 24, 10, 6, 200, 3, 2),     # 5x3 output: not a multiple of any pixel box
    (3, 64, 13, 11, 72, 3, 1),
    (2, 40, 14, 10, 200, 1, 2),
    (3, 16, 6, 14, 72, 3, 2),
]


def _conv_lib():
    from distributed_torch_horovod_gcp_b200.ops import conv, kernels
    assert kernels.has("conv_implicit_gemm"), "conv kernel missing from libb200dp_kernels.so"
    return conv._lib


@gpu
@pytest.mark.parametrize("N,Cin,H,W,Cout,R,stride", CONV_CASES)
def test_conv_fprop_dgrad_vs_fp64(N, Cin, H, W, Cout, R, stride):
    lib = _conv_lib()
    g = torch.Generator(device="cuda").manual_seed(N * H * W + Cin + Cout)
    pad = (R - 1) // 2
    OH, OW = H // stride, W // stride
    x = _nhwc(torch.randn(N, Cin, H, W, device="cuda", generator=g))
    w = _nhwc(torch.randn(Cout, Cin, R, R, device="cuda", generator=g) * (Cin * R * R) ** -0.5)
    dy = _nhwc(torch.randn(N, Cout, OH, OW, device="cuda", generator=g))
    y64, ym = conv_fprop_ref(x, w, stride, pad)
    yb = conv_bound(y64, ym, R * R * _pad64(Cin))
    dx64, dxm = conv_dgrad_ref(dy, w, x.shape, stride, pad)
    dxb = conv_bound(dx64, dxm, R * R * _pad64(Cout))
    first = None
    for bn in (64, 128):
        y = _nan_nhwc(N, Cout, OH, OW)
        assert lib.b200dp_conv_fprop(x.data_ptr(), w.data_ptr(), y.data_ptr(), N, H, W, Cin, Cout, R, R, stride,
                                     pad, bn, 0, None, _stream()) == 0, lib.b200dp_conv_last_error()
        dx = _nan_nhwc(N, Cin, H, W)
        assert lib.b200dp_conv_dgrad(dy.data_ptr(), w.data_ptr(), dx.data_ptr(), N, H, W, Cin, Cout, R, R, stride,
                                     pad, bn, 0, _stream()) == 0, lib.b200dp_conv_last_error()
        torch.cuda.synchronize()
        _check_split(y, y64, yb, "conv fprop")
        _check_split(dx, dx64, dxb, "conv dgrad")
        if stride == 2:
            for ph in (0, 1):
                for pw in (0, 1):
                    sl = (slice(None), slice(None), slice(ph, None, 2), slice(pw, None, 2))
                    if R == 1 and (ph or pw):       # no tap reaches these positions
                        assert bool((dx[sl] == 0).all()), f"1x1 s2 dgrad: parity ({ph}, {pw}) not zero"
                        assert float(dx64[sl].abs().max()) == 0.0
                    else:
                        assert float(dx64[sl].abs().max()) > 0.0
                        _check(dx[sl], dx64[sl], dxb[sl], "conv dgrad s2 parity classes")
        if first is None:
            first = (y, dx)
        else:
            assert torch.equal(y, first[0]) and torch.equal(dx, first[1])


# ================================================================================================ BatchNorm
BN_EPS = 1e-5
BN_MOM = 0.1


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def standalone_depth(M, C, sms):
    """Longest addition chain of ``bn_stats_kernel`` / ``bn_bwd_reduce_kernel`` (grid G = min(SMs, 256) blocks of
    1024 threads, a thread owning one 8-channel group): its serial chain over ceil(M C / 8 / (1024 G)) vectors, the
    block's sum over the 1024 / (C / 8) threads of a group, the last block's sum of G slots, and the add into the
    zeroed output.  Vectors are dealt to the lowest threads and blocks first, and adding the zero partials of idle
    threads / blocks is exact, so only min(groups, M) partials of a block and the slots of the
    ceil(M C / 8 / 1024) blocks with data count."""
    G = min(sms, 256)
    V = C // 8
    nvec = M * V
    return _cdiv(nvec, 1024 * G) + min(1024 // V, M) + min(G, _cdiv(nvec, 1024)) + 1


def _choose_box(W, H, N, rows):
    """conv_sm90.cu choose_box: the {bw, bh, bn} pixel box of an M tile."""
    best, box = 1e30, (1, 1, rows)
    w = 1
    while w <= rows:
        h = 1
        while w * h <= rows:
            n = rows // (w * h)
            covered = (_cdiv(W, w) * w) * (_cdiv(H, h) * h) * (_cdiv(N, n) * n)
            score = covered - 1e-3 * w - 1e-6 * h
            if score < best:
                best, box = score, (w, h, n)
            h <<= 1
        w <<= 1
    return box


def epilogue_depth(items, sms):
    """Longest addition chain of the GEMM / convolution epilogue statistics (``store_slab``, ``stats_flush``,
    ``stats_finalize``) over ``items`` output tiles on G = min(items, SMs) persistent CTAs (CTA b takes tiles
    b, b + G, ...: at most T = ceil(items / G) each): 32 rows of a slab in a lane's registers, at most one add per
    slab (4 per tile) into a warp's private accumulator and at most one flush per slab into the CTA's slot, the 4
    lane-quarter regions, the last CTA's sum of G slots, and the add into the zeroed accumulator."""
    G = min(items, sms, 256)
    return 32 + 2 * 4 * _cdiv(items, G) + 4 + G + 1


def _sig_bits(v):
    """Significant bits of each value of a float64 tensor (0 for 0)."""
    m, _ = torch.frexp(v.abs())
    bits = torch.zeros_like(v, dtype=torch.int64)
    for b in range(1, 54):
        done = (bits == 0) & (torch.ldexp(m, torch.full_like(bits, b)) == torch.ldexp(m, torch.full_like(bits, b)).round())
        bits[done] = b
    return torch.where(v == 0, torch.zeros_like(bits), bits)


def bn_stat_bounds(x2, D, eps=BN_EPS):
    """mean / variance / invstd as ``bn_finalize`` computes them from sums with chain depth D, for [M, C] x2:
    S1, S2 within 1.01 D u sum|x|, sum x^2; m~ = fl(S1 / M): Em = 1.01 D u mean|x| + 1.01 u |m|;
    fl(S2 / M) within Eq = 1.01 (D + 1) u E[x^2];  var~ = fl(fl(S2/M) - fl(m~ m~)) (or one fma), clamped at 0:
    Evar = (Eq + Em (2|m| + Em) + u (|m| + Em)^2 + u var) / (1 - u) -- the cancellation term is Eq + 2|m| Em;
    invstd = rsqrtf(fl(var~ + fl32(eps))): nu = (Evar + u (var + eps + Evar) + u eps) / (var + eps) and
    rho = (1 - nu)^-1/2 (1 + U_RSQRT) - 1.
    A constant channel of value v with b significant bits is exact when every partial sum k v, k v^2 (k <= M) is
    an fp32 number, i.e. 2 b + bits(M) <= 24: then S1 = M v, S2 = M v^2, m~ = v and var~ = 0, so Em = Evar = 0.
    (With 8-bit bf16 values that holds up to M = 256; beyond it a constant channel can get var~ of a few u v^2
    instead of 0, and invstd = rsqrt(eps) only if eps dominates that.  Dead post-ReLU channels, v = 0, are exact.)"""
    x = x2.double()
    M = x.shape[0]
    # divided on the CPU: a CUDA division by a scalar multiplies by its reciprocal, which would make the mean of
    # a constant channel inexact
    m = (x.sum(0).cpu() / M).to(x.device)
    var = ((x - m) ** 2).sum(0).cpu().div(M).to(x.device)
    q = (x * x).sum(0).cpu().div(M).to(x.device)
    Em = 1.01 * D * U32 * x.abs().mean(0) + 1.01 * U32 * m.abs()
    Eq = 1.01 * (D + 1) * U32 * q
    Evar = (Eq + Em * (2 * m.abs() + Em) + U32 * (m.abs() + Em) ** 2 + U32 * var) / (1 - U32)
    exact = (x == x[:1]).all(0) & (2 * _sig_bits(x[0]) + M.bit_length() <= 24)
    Em = torch.where(exact, torch.zeros_like(Em), Em)
    Evar = torch.where(exact, torch.zeros_like(Evar), Evar)
    nu = (Evar + U32 * (var + eps + Evar) + U32 * eps) / (var + eps)
    assert float(nu.max()) < 0.5, "the variance bound is too loose for the invstd bound to apply"
    rho = (1 - nu) ** -0.5 * (1 + U_RSQRT) - 1
    r = 1 / torch.sqrt(var + eps)
    return m, var, r, Em, Evar, rho


def bn_fwd_bounds(x2, gamma, beta, res2, relu, D, eps=BN_EPS):
    """y of the training forward: a = fl(g is), b = fl(beta - fl(fl(m~ g) is)), y = bf16(relu(fl(fma(x, a, b)) + r)).
    Against y* = g r* (x - m*) + beta (+ res):
    E_lin = |g| r* rho |x - m*| + |g| r* (1 + rho) Em + (1 + rho) r* |g| u (|x| + 3.03 (|m*| + Em)) + u |beta|,
    the fma and the residual add one rounding each, ReLU is 1-Lipschitz, then the bf16 store.  Also returns the
    pre-ReLU reference and its bound (for the mask bits)."""
    m, var, r, Em, Evar, rho = bn_stat_bounds(x2, D, eps)
    x = x2.double()
    g, b = gamma.double(), beta.double()
    y = g * r * (x - m) + b
    E = g.abs() * r * rho * (x - m).abs() + g.abs() * r * (1 + rho) * Em \
        + (1 + rho) * r * g.abs() * U32 * (x.abs() + 3.03 * (m.abs() + Em)) + U32 * b.abs()
    E = E + U32 * (y.abs() + E)
    if res2 is not None:
        y = y + res2.double()
        E = E + U32 * (y.abs() + E)
    pre, Epre = y, E
    if relu:
        y = y.clamp_min(0)
    return y, bf16_store(E, y), pre, Epre


def bn_bwd_bounds(x2, dz2, gamma, D_f, D_b, pbf16, eps=BN_EPS):
    """dx, dgamma, dbeta of the backward at the batch statistics of x, for dz = dy masked by the ReLU bits.
    The kernel reuses the forward's m~, is (bounds of ``bn_stat_bounds`` with depth D_f); its sums have depth D_b:
    S1 = sum dz within E1 = 1.01 D_b u sum|dz|; S2 = sum dz fl(x - m~) within
    EP = 1.01 (D_b + 1) u sum |dz| (|x - m*| + Em) + Em |S1*| of P* = sum dz (x - m*).
    dbeta = S1 (E1); dgamma = fl(S2 is) within EP r*(1 + rho) + |P*| r* rho + u |dgamma|; bf16 params: a store.
    dx = bf16(fl(a fl(dz - k1 - xhat k2))), k1 = fl(S1 fl(1/M)), k2 = fl(fl(S2 is) fl(1/M)), xhat = fl(fl(x - m~) is):
    E_k1 = E1/M + 2.02 u |k1*|, E_k2 = (EP r*(1+rho) + |P*| r* rho) / M + 3.03 u (|k2*| + ...),
    E_xh = r* (1 + rho) Em + rho |xhat*| + 2.02 u (1 + rho) |xhat*|, the two roundings of the difference
    (2.02 u of its terms), a within (rho + u) of g r*, and one rounding of the product."""
    m, var, r, Em, Evar, rho = bn_stat_bounds(x2, D_f, eps)
    x, dz, g = x2.double(), dz2.double(), gamma.double()
    M = x.shape[0]
    xc = x - m
    xh = xc * r
    S1 = dz.sum(0)
    P = (dz * xc).sum(0)
    E1 = 1.01 * D_b * U32 * dz.abs().sum(0)
    EP = 1.01 * (D_b + 1) * U32 * (dz.abs() * (xc.abs() + Em)).sum(0) + Em * S1.abs()
    db, dbb = S1, E1
    dg = P * r
    dgb = EP * r * (1 + rho) + P.abs() * r * rho
    dgb = dgb + U32 * (dg.abs() + dgb)
    if pbf16:
        dbb, dgb = bf16_store(dbb, db), bf16_store(dgb, dg)
    k1, k2 = S1 / M, P * r / M
    Ek1 = E1 / M + 2.02 * U32 * (k1.abs() + E1 / M)
    Ek2 = (EP * r * (1 + rho) + P.abs() * r * rho) / M
    Ek2 = Ek2 + 3.03 * U32 * (k2.abs() + Ek2)
    Exh = r * (1 + rho) * Em + rho * xh.abs() + 2.02 * U32 * (1 + rho) * (xh.abs() + r * Em)
    t = dz - k1 - xh * k2
    Et = Ek1 + xh.abs() * Ek2 + Exh * (k2.abs() + Ek2) \
        + 2.02 * U32 * (dz.abs() + k1.abs() + Ek1 + (xh.abs() + Exh) * (k2.abs() + Ek2))
    dx = g * r * t
    ra = (1 + rho) * (1 + U32)
    dxb = g.abs() * r * (ra * Et + (ra - 1) * t.abs())
    dxb = dxb + U32 * (dx.abs() + dxb)
    return (dx, bf16_store(dxb, dx)), (dg, dgb), (db, dbb)


def running_stats_bounds(rm0, rv0, m, var, Em, Evar, M, mom, pbf16):
    """running_mean / running_var after one step of ``bn_finalize_kernel`` over M rows: fl((1 - mom) r + mom s) in
    fp32, s = m~ or the unbiased var~ M / max(M - 1, 1), then the store in the parameter dtype.  Against the float64
    update of rm0 / rv0 with the exact statistics: the error of s times mom, and 5 u of the terms for fl32(mom), the
    two products and the sum.  Returns (rm, Erm, rv, Erv)."""
    c = M / max(M - 1, 1)
    rm = (1 - mom) * rm0 + mom * m
    Erm = mom * Em * (1 + U32) + 5 * U32 * ((1 - mom) * rm0.abs() + mom * (m.abs() + Em))
    rv = (1 - mom) * rv0 + mom * var * c
    Eunb = c * (Evar + 2.02 * U32 * (var + Evar))
    Erv = mom * Eunb * (1 + U32) + 5 * U32 * ((1 - mom) * rv0.abs() + mom * (var * c + Eunb))
    if pbf16:
        Erm, Erv = bf16_store(Erm, rm), bf16_store(Erv, rv)
    return rm, Erm, rv, Erv


def bn_inputs(M, C, seed, D=0):
    """x [M, C]: per channel, c % 4 == 0: zero mean; 1: |mean| / std = 8; 2: |mean| / std = 64; 3: constant
    (var = 0, invstd = rsqrt(eps)) of a value with at most 4 significant bits, 0 included (a dead ReLU channel);
    std in (0.5, 2) and the sign of the mean alternating.  The worst-case variance bound of depth D is informative
    (nu < 1/2 in ``bn_stat_bounds``) for |mean| / std = 64 only while 3.03 D u 64^2 < 1/4, D < 339: deeper
    reductions (C = 8: 1024 threads per channel group in a block) take |mean| / std = 16 in that slot."""
    g = torch.Generator().manual_seed(seed)
    std = torch.rand(C, generator=g) * 1.5 + 0.5
    sign = torch.where(torch.arange(C) % 8 < 4, 1.0, -1.0)
    big = 64.0 if 3.03 * D * U32 * 64.0 ** 2 < 0.25 else 16.0
    ratio = torch.tensor([0.0, 8.0, big, 0.0]).repeat(C // 4 + 1)[:C]
    x = torch.randn(M, C, generator=g) * std + sign * ratio * std
    const = torch.arange(C) % 4 == 3
    vals = torch.tensor([0.0, 1.5, -3.0, 0.75, -6.5, 2.0]).repeat(C // 6 + 1)[:C]
    x[:, const] = vals[const]
    return x.bfloat16()


def _bn_module(C, pdtype, seed):
    g = torch.Generator().manual_seed(seed)
    bn = torch.nn.BatchNorm2d(C, eps=BN_EPS, momentum=BN_MOM)
    with torch.no_grad():
        bn.weight.copy_(torch.rand(C, generator=g) + 0.5)
        bn.bias.copy_(0.3 * torch.randn(C, generator=g))
        bn.running_mean.copy_(torch.randn(C, generator=g))
        bn.running_var.copy_(torch.rand(C, generator=g) + 0.5)
    return bn.cuda().to(pdtype)


def _bits_to_mask(bits, M, C):
    return ((bits.view(M, C // 8, 1) >> torch.arange(8, device=bits.device, dtype=torch.uint8)) & 1).view(M, C).bool()


def _shape4(M):
    return {1: (1, 1, 1), 7: (1, 7, 1), 1000: (10, 10, 10), 8 * 56 * 56: (8, 56, 56)}[M]


# C, M, stats source, param dtype, residual, relu
BN_CASES = [
    (8, 1, "standalone", torch.bfloat16, False, True),
    (8, 1000, "gemm", torch.float32, True, True),
    (8, 7, "standalone", torch.float32, True, False),
    (64, 7, "conv", torch.bfloat16, True, True),
    (64, 8 * 56 * 56, "standalone", torch.bfloat16, True, True),
    (64, 8 * 56 * 56, "gemm", torch.float32, False, True),
    (256, 1000, "standalone", torch.float32, False, True),
    (256, 8 * 56 * 56, "conv", torch.bfloat16, False, False),
    (256, 1, "gemm", torch.bfloat16, False, False),
    (1024, 7, "gemm", torch.float32, True, True),
    (2048, 1000, "standalone", torch.bfloat16, True, False),
    (2048, 7, "standalone", torch.float32, False, True),
    (2048, 1000, "gemm", torch.bfloat16, True, True),
    (128, 1000, "conv", torch.float32, True, True),
]


def _run_bn_train(x, bn, res, relu, src):
    """The training forward with statistics from the stand-alone pass, or from the epilogue of a 1x1 (GEMM) or 3x3
    (implicit-GEMM) convolution whose weights pass x through unchanged (y = bf16(x * 1) = x), as conv_bn_act runs
    it.  Returns the BN output, its mask bits, the saved (mean, invstd, a), and the depth of the statistics sums."""
    from distributed_torch_horovod_gcp_b200.ops import bn as B, conv as CV
    N, C, H, W = x.shape
    M = N * H * W
    if src == "standalone":
        return B.bn_forward(x, bn, res, relu)
    R = 1 if src == "gemm" else 3
    conv = torch.nn.Conv2d(C, C, R, 1, R // 2, bias=False).cuda().to(torch.bfloat16)
    with torch.no_grad():
        conv.weight.zero_()
        conv.weight[:, :, R // 2, R // 2] = torch.eye(C, device="cuda")
    conv = conv.to(memory_format=torch.channels_last)
    conv.weight.requires_grad_(False)
    stats = B.fused_stats(bn, C, x.device)
    assert stats is not None
    before = stats.clone()
    assert CV.kind(x, conv) == ("gemm" if src == "gemm" else "implicit")
    y0 = CV.conv2d(x, conv, stats=stats)
    assert bool((stats != before).any() or M == 0)
    assert torch.equal(y0, x), "pass-through convolution changed its input"
    y, mask, ws = B.bn_forward(y0.contiguous(memory_format=torch.channels_last), bn, res, relu, stats_in=stats)
    assert float(stats.abs().max()) == 0.0, "bn_finalize did not re-zero the epilogue accumulator"
    return y, mask, ws


def stats_depth(src, N, C, H, W):
    """Depth of the statistics sums for ``_run_bn_train``: the pass-through convolution's output tiles are
    128-row M tiles (GEMM) or {bw, bh, bn} pixel boxes (implicit GEMM) times ceil(C / BN), BN = 64 for C <= 64
    else 128 (``pick_bn``)."""
    M = N * H * W
    if src == "standalone":
        return standalone_depth(M, C, _sms())
    if src == "gemm":
        tiles = _cdiv(M, 128)
    else:
        bw, bh, bnn = _choose_box(W, H, N, 128)
        tiles = _cdiv(W, bw) * _cdiv(H, bh) * _cdiv(N, bnn)
    return epilogue_depth(tiles * _cdiv(C, 64 if C <= 64 else 128), _sms())


def _to2(t):
    return t.permute(0, 2, 3, 1).reshape(-1, t.shape[1])


@gpu
@pytest.mark.parametrize("C,M,src,pdtype,with_res,relu", BN_CASES)
def test_bn_train_fwd_bwd_vs_fp64(C, M, src, pdtype, with_res, relu):
    from distributed_torch_horovod_gcp_b200.ops import bn as B
    if src == "conv" and C < 16:
        pytest.skip("the implicit-GEMM convolution needs Cin >= 16")
    N, H, W = _shape4(M)
    D = stats_depth(src, N, C, H, W)
    x2 = bn_inputs(M, C, seed=C + M, D=max(D, standalone_depth(M, C, _sms())))
    x = x2.view(N, H, W, C).permute(0, 3, 1, 2).cuda().contiguous(memory_format=torch.channels_last)
    g = torch.Generator().manual_seed(C * 3 + M)
    res2 = torch.randn(M, C, generator=g).bfloat16() if with_res else None
    res = res2.view(N, H, W, C).permute(0, 3, 1, 2).cuda().contiguous(memory_format=torch.channels_last) \
        if with_res else None
    bn = _bn_module(C, pdtype, seed=C + 1)
    rm0, rv0 = bn.running_mean.double().clone(), bn.running_var.double().clone()
    nbt0 = int(bn.num_batches_tracked)
    y, mask, ws = _run_bn_train(x, bn, res, relu, src)
    torch.cuda.synchronize()
    x2c = x2.cuda()
    tag = f"{src} stats"
    m, var, r, Em, Evar, rho = bn_stat_bounds(x2c, D)
    _check(ws[0], m, Em, f"bn mean ({tag})")
    _check(ws[1], r, rho * r, f"bn invstd ({tag})")
    yr, yb, pre, Epre = bn_fwd_bounds(x2c, bn.weight.detach(), bn.bias.detach(), res2.cuda() if with_res else None,
                                      relu, D)
    _check(_to2(y), yr, yb, f"bn fwd y ({tag})")
    if relu:
        bits = _bits_to_mask(mask, M, C)
        sure = pre.abs() > Epre
        assert bool((bits[sure] == (pre[sure] > 0)).all()), "ReLU mask bit disagrees with the sign of y"
        assert bool((_to2(y)[~bits] == 0).all()), "y nonzero where the mask bit is clear"
    # running statistics (param dtype), momentum 0.1, unbiased variance
    rm, Erm, rv, Erv = running_stats_bounds(rm0, rv0, m, var, Em, Evar, M, BN_MOM, pdtype == torch.bfloat16)
    _check(bn.running_mean, rm, Erm, "bn running_mean")
    _check(bn.running_var, rv, Erv, "bn running_var (unbiased)")
    assert int(bn.num_batches_tracked) == nbt0 + 1
    # backward, with and without the mask
    dy2 = torch.randn(M, C, generator=g).bfloat16() + 0.25
    dy = dy2.view(N, H, W, C).permute(0, 3, 1, 2).cuda().contiguous(memory_format=torch.channels_last)
    for use_mask in ((False, True) if relu else (False,)):
        mk = mask if use_mask else None
        dx, dgam, dbet, dres = B.bn_backward(dy, bn, x, mk, ws, write_dres=True)
        torch.cuda.synchronize()
        dz2 = dy2.cuda() * _bits_to_mask(mask, M, C).bfloat16() if use_mask else dy2.cuda()
        (dxr, dxb), (dgr, dgb), (dbr, dbb) = bn_bwd_bounds(x2c, dz2, bn.weight.detach(), D,
                                                           standalone_depth(M, C, _sms()),
                                                           pdtype == torch.bfloat16)
        t2 = f"{'masked' if use_mask else 'no mask'}"
        _check(_to2(dx), dxr, dxb, f"bn bwd dx ({t2})")
        assert dgam.dtype == pdtype and dbet.dtype == pdtype
        _check(dgam, dgr, dgb, "bn bwd dgamma")
        _check(dbet, dbr, dbb, "bn bwd dbeta")
        assert torch.equal(_to2(dres), dz2), "dres is not the masked dy"


@gpu
@pytest.mark.parametrize("pdtype", [torch.bfloat16, torch.float32], ids=["bf16", "fp32"])
@pytest.mark.parametrize("with_res,relu", [(False, False), (True, True), (False, True)])
def test_bn_inference_apply_vs_fp64(pdtype, with_res, relu):
    """Frozen statistics: a = fl(g fl(rsqrt(fl(rv + eps)))) and b = fl(beta - fl(rm a)) in torch fp32 (rsqrt within
    U_RSQRT), then y = bf16(relu(fl(fma(x, a, b)) + r)).  Against y* = g (x - rm) / sqrt(rv + eps) + beta:
    a within rho_a = 1.01 (U_RSQRT + 3u) of g r*, E_b = |rm| |a*| (rho_a + u) + u |beta - rm a*|, the fma and the
    residual add one rounding each."""
    from distributed_torch_horovod_gcp_b200.ops import bn as B
    C, (N, H, W) = 256, _shape4(1000)
    M = N * H * W
    x2 = bn_inputs(M, C, seed=5)
    x = x2.view(N, H, W, C).permute(0, 3, 1, 2).cuda().contiguous(memory_format=torch.channels_last)
    g = torch.Generator().manual_seed(6)
    res2 = torch.randn(M, C, generator=g).bfloat16() if with_res else None
    res = res2.view(N, H, W, C).permute(0, 3, 1, 2).cuda().contiguous(memory_format=torch.channels_last) \
        if with_res else None
    bn = _bn_module(C, pdtype, seed=7).eval()
    with torch.no_grad():
        bn.running_mean.copy_(x2.double().mean(0).to(pdtype))
        bn.running_var.copy_((x2.double().var(0) + 0.01).to(pdtype))
    y = B.bn_act(x, bn, relu, res)
    torch.cuda.synchronize()
    xd = x2.cuda().double()
    gm, bt = bn.weight.detach().double(), bn.bias.detach().double()
    rm, rv = bn.running_mean.double(), bn.running_var.double()
    r = 1 / torch.sqrt(rv + BN_EPS)
    a = gm * r
    ra = 1.01 * (U_RSQRT + 3 * U32)
    yr = a * (xd - rm) + bt
    Eb = rm.abs() * a.abs() * (ra + U32) * 1.01 + U32 * (bt - rm * a).abs() * 1.01
    E = xd.abs() * a.abs() * ra + Eb
    E = E + U32 * (yr.abs() + E)
    if with_res:
        yr = yr + res2.cuda().double()
        E = E + U32 * (yr.abs() + E)
    if relu:
        yr = yr.clamp_min(0)
    _check(_to2(y), yr, bf16_store(E, yr), "bn inference apply")


@gpu
def test_bn_one_pass_variance_vs_library():
    """|mean| / std = 8 at M = 8*56*56, C = 64, both statistics sources: the kernel's BatchNorm output must be
    within twice the error of ``nn.BatchNorm2d`` in bf16 on the same input (both against float64), or within one
    bf16 rounding (2^-8).  The 64 regime is printed for the record."""
    from distributed_torch_horovod_gcp_b200.ops import bn as B
    C, M = 64, 8 * 56 * 56
    N, H, W = _shape4(M)
    for ratio in (8.0, 64.0):
        g = torch.Generator().manual_seed(int(ratio))
        std = torch.rand(C, generator=g) + 0.5
        x2 = (torch.randn(M, C, generator=g) * std + ratio * std).bfloat16()
        x = x2.view(N, H, W, C).permute(0, 3, 1, 2).cuda().contiguous(memory_format=torch.channels_last)
        ref = None
        for src in ("standalone", "gemm"):
            bn = _bn_module(C, torch.bfloat16, seed=3)
            lib_bn = _bn_module(C, torch.bfloat16, seed=3)
            y, _, _ = _run_bn_train(x, bn, None, False, src)
            y_lib = lib_bn(x)
            torch.cuda.synchronize()
            xd = x2.cuda().double()
            m, v = xd.mean(0), xd.var(0, unbiased=False)
            ref = (xd - m) / torch.sqrt(v + BN_EPS) * bn.weight.double() + bn.bias.double()
            e_k = float((_to2(y).double() - ref).norm() / ref.norm())
            e_l = float((_to2(y_lib).double() - ref).norm() / ref.norm())
            print(f"\n[bn one-pass] |mean|/std={ratio:g} {src}: kernel {e_k:.3e} nn.BatchNorm2d bf16 {e_l:.3e}", end="")
            if ratio == 8.0:
                assert e_k <= max(2 * e_l, U_BF16), (src, e_k, e_l)
    print()


# ================================================================================================ pooling and stem
def _bn_lib():
    from distributed_torch_horovod_gcp_b200.ops import bn, kernels
    assert kernels.has("max_pool_3x3_s2") and kernels.has("global_avg_pool") and kernels.has("stem_conv")
    return bn._lib


def maxpool_ref(x):
    """float64 3x3 / stride 2 / pad 1 max-pool of [N, C, H, W] x: the max, the tap (kh * 3 + kw) of the FIRST
    maximum in scan order (torch.argmax returns the first), the padding never chosen."""
    N, C, H, W = x.shape
    OH, OW = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    xp = F.pad(x.double(), (1, 2 * OW - W, 1, 2 * OH - H), value=float("-inf"))
    cols = F.unfold(xp, 3, stride=2).view(N, C, 9, OH * OW)
    val, arg = cols.max(2)[0], cols.argmax(2)
    return val.view(N, C, OH, OW), arg.view(N, C, OH, OW)


def maxpool_bwd_ref(dy, arg, x_shape):
    """float64 scatter of dy to the arg-max taps, the same on |dy|, and the number of terms per input element."""
    N, C, H, W = x_shape
    OH, OW = dy.shape[2], dy.shape[3]
    Hp, Wp = 2 * OH + 1, 2 * OW + 1
    outs = []
    for v in (dy.double(), dy.double().abs(), torch.ones_like(dy, dtype=torch.float64)):
        cols = torch.zeros(N, C, 9, OH * OW, dtype=torch.float64, device=dy.device)
        cols.scatter_(2, arg.view(N, C, 1, OH * OW), v.reshape(N, C, 1, OH * OW))
        full = F.fold(cols.view(N, C * 9, OH * OW), (Hp, Wp), 3, stride=2)
        outs.append(full[:, :, 1:H + 1, 1:W + 1])
    return outs


def maxpool_inputs(N, C, H, W, seed):
    """Forced ties: post-ReLU values on a grid of 1/2 (many all-zero windows and equal maxima), and whole rows of
    one value."""
    g = torch.Generator().manual_seed(seed)
    x = (torch.randn(N, C, H, W, generator=g) * 2).round().clamp_min(0) / 2
    x[:, :, ::3] = 1.5
    return x


MAXPOOL_SHAPES = [(2, 64, 8, 8), (3, 16, 10, 14), (1, 8, 2, 2), (2, 24, 9, 9), (2, 16, 7, 10), (2, 8, 1, 1),
                  (2, 64, 112, 112)]


@gpu
@pytest.mark.parametrize("shape", MAXPOOL_SHAPES, ids=lambda s: "x".join(map(str, s)))
def test_maxpool_vs_fp64(shape):
    """Forward: the max bit for bit and the first arg-max.  Backward: the 2x2-patch kernel (H, W even) adds the
    k <= 4 contributions of an input element in bf16 (k - 1 bf16 roundings of partial sums); the generic kernel in
    fp32, then one bf16 store."""
    lib = _bn_lib()
    N, C, H, W = shape
    OH, OW = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    x = _nhwc(maxpool_inputs(N, C, H, W, seed=H * W + C).cuda())
    y = torch.empty(N, C, OH, OW, device="cuda", dtype=torch.bfloat16, memory_format=torch.channels_last)
    idx = torch.empty(N * OH * OW * C, device="cuda", dtype=torch.uint8)
    assert lib.b200dp_maxpool_fwd(x.data_ptr(), y.data_ptr(), idx.data_ptr(), N, H, W, C, _stream()) == 0
    torch.cuda.synchronize()
    val, arg = maxpool_ref(x)
    assert torch.equal(y.double(), val), "max-pool value differs from the float64 max"
    ties = (F.unfold(F.pad(x.double(), (1, 2 * OW - W, 1, 2 * OH - H), value=float("-inf")), 3, stride=2)
            .view(N, C, 9, -1) == val.view(N, C, 1, -1)).sum(2)
    assert H * W == 1 or int((ties > 1).sum()) > 0, "no ties: the arg-max check is vacuous"
    k_arg = idx.view(N, OH, OW, C).permute(0, 3, 1, 2).long()
    bad = k_arg != arg
    assert not bool(bad.any()), f"{int(bad.sum())} arg-max taps are not the first maximum"
    dy = _nhwc(torch.randn(N, C, OH, OW, device="cuda"))
    dx = _nan_nhwc(N, C, H, W)
    assert lib.b200dp_maxpool_bwd(dy.data_ptr(), idx.data_ptr(), dx.data_ptr(), N, H, W, C, _stream()) == 0
    torch.cuda.synchronize()
    ref, mag, cnt = maxpool_bwd_ref(dy, arg, x.shape)
    assert float(cnt.max()) <= 4
    if H % 2 == 0 and W % 2 == 0:
        _check(dx, ref, ((1 + U_BF16) ** (cnt - 1).clamp_min(0) - 1) * mag, "maxpool bwd 2x2-patch (bf16 adds)")
    else:
        _check(dx, ref, bf16_store(1.01 * (cnt - 1).clamp_min(0) * U32 * mag, ref), "maxpool bwd generic (fp32)")


@gpu
@pytest.mark.parametrize("N,C,H,W", [(4, 64, 7, 7), (3, 16, 1, 1), (2, 256, 14, 14), (5, 2048, 7, 7)])
def test_avgpool_vs_fp64(N, C, H, W):
    """Forward: fp32 sum of HW terms (HW additions from 0), times fl(1/HW), bf16 store:
    E = 1.01 HW u mean|x| (1 + 2.02 u) + 2.02 u |mean|.  Backward: bf16(fl(dy fl(1/HW))): E = 2.02 u |dy / HW|."""
    lib = _bn_lib()
    HW = H * W
    g = torch.Generator(device="cuda").manual_seed(N + C + HW)
    x = _nhwc(torch.randn(N, C, H, W, device="cuda", generator=g) + 1.0)
    y = torch.empty(N, C, device="cuda", dtype=torch.bfloat16)
    assert lib.b200dp_avgpool_fwd(x.data_ptr(), y.data_ptr(), N, HW, C, _stream()) == 0
    dy = torch.randn(N, C, device="cuda", generator=g).bfloat16()
    dx = torch.empty(N, C, H, W, device="cuda", dtype=torch.bfloat16, memory_format=torch.channels_last)
    assert lib.b200dp_avgpool_bwd(dy.data_ptr(), dx.data_ptr(), N, HW, C, _stream()) == 0
    torch.cuda.synchronize()
    xd = x.double()
    ref = xd.mean((2, 3))
    E = 1.01 * HW * U32 * xd.abs().mean((2, 3)) * (1 + 2.02 * U32) + 2.02 * U32 * ref.abs()
    _check(y, ref, bf16_store(E, ref), "avgpool fwd")
    dref = (dy.double() / HW)[:, :, None, None].expand(N, C, H, W)
    _check(dx, dref, bf16_store(2.02 * U32 * dref.abs(), dref), "avgpool bwd")


@gpu
@pytest.mark.parametrize("N,H,W", [(1, 2, 8), (2, 4, 224), (3, 16, 24)])
def test_stem_im2col_and_gemm_vs_fp64(N, H, W):
    """im2col: columns kh * 24 + kw * 3 + c (kw * 3 + c < 21) equal the unfold of the zero-padded input bit for
    bit.  Output: a GEMM over 168 columns (three zero-weighted per kernel row, K zero-filled to 192), bf16 store.
    Weight gradient: split-K fp32 sums of 64 ceil(M / 64) products per split, s splits added to a zeroed buffer,
    then one bf16 rounding."""
    from distributed_torch_horovod_gcp_b200.ops import conv as CV, gemm as G
    lib = _bn_lib()
    g = torch.Generator(device="cuda").manual_seed(N * H * W)
    x = _nhwc(torch.randn(N, 3, H, W, device="cuda", generator=g))
    OH, OW = H // 2, W // 2
    M = N * OH * OW
    cols = torch.empty(M, CV.STEM_KP, device="cuda", dtype=torch.bfloat16)
    assert lib.b200dp_stem_im2col(x.data_ptr(), cols.data_ptr(), N, H, W, _stream()) == 0
    torch.cuda.synchronize()
    ref = F.unfold(x.float(), 7, padding=3, stride=2).view(N, 3, 7, 7, OH * OW)      # [n, c, kh, kw, l]
    ref = ref.permute(0, 4, 2, 3, 1).reshape(M, 7, 21).bfloat16()
    assert torch.equal(cols.view(M, 7, 24)[:, :, :21], ref), "stem im2col differs from unfold"
    w = _nhwc(torch.randn(64, 3, 7, 7, device="cuda", generator=g) * 0.1).requires_grad_(True)
    y = CV._ConvFn.apply(x, w, "stem", 2, 3)
    dy = torch.randn(y.shape, device="cuda", generator=g).bfloat16()
    y.backward(dy)
    torch.cuda.synchronize()
    y64, ym = conv_fprop_ref(x, w.detach(), 2, 3)
    _check(y, y64, conv_bound(y64, ym, 192 // 64 * 64), "stem fprop")
    gw = torch.nn.grad.conv2d_weight
    dw64 = gw(x.double(), w.shape, dy.double(), 2, 3)
    dwm = gw(x.double().abs(), w.shape, dy.double().abs(), 2, 3)
    s = G._splits_for(64, CV.STEM_KP, M)
    _check(w.grad, dw64, bf16_store(2 * (_pad64(M) + s + 1) * U32 * dwm, dw64), "stem wgrad")


# ================================================================================================ CPU self-checks
def _must_fail(fn):
    with pytest.raises(AssertionError):
        fn()
    fp64_bounds._WORST.pop("perturbed", None)


def _perturb_tightest(got, ref, bound):
    """got moved by 3 bf16 ulps of the reference at the (nonzero) element whose bound is tightest relative to it."""
    rel = bound.reshape(-1) / ref.abs().reshape(-1)
    i = int(torch.argmin(torch.where(ref.reshape(-1) != 0, rel, torch.full_like(rel, float("inf")))))
    bad = got.double().clone().reshape(-1)
    bad[i] += 3 * 2.0 ** -7 * float(ref.reshape(-1)[i].abs())
    return bad.view_as(got)


def _accept_reject(got32, ref, bound):
    _check(got32, ref, bound, "cpu self-check")
    _must_fail(lambda: _check(_perturb_tightest(got32, ref, bound), ref, bound, "perturbed"))


def test_fast_erf_bound_covers_an_fp32_emulation():
    """fast_erf evaluated in float32 with exact exp (the CUDA intrinsics are within the bound's U_DIV / U_EX2 of
    these), over every 2^-10 step of (-8, 8): inside ``fast_erf_err``; A&S alone is 1.5e-7 from erf."""
    x = torch.arange(-8 * 1024, 8 * 1024 + 1, dtype=torch.float32) / 1024
    ax = x.abs()
    t = 1.0 / (0.3275911 * ax + 1.0)
    poly = ((((1.061405429 * t - 1.453152027) * t + 1.421413741) * t - 0.284496736) * t + 0.254829592)
    y = torch.copysign(1.0 - poly * t * torch.exp(-ax * ax), x)
    err = (y.double() - torch.erf(x.double())).abs()
    assert bool((err <= fast_erf_err(x.double())).all())


def test_gemm_bounds_accept_fp32_and_reject_perturbed():
    for path in ("plain", "res_only_cancel", "bias_f32_alpha_relu_res", "gelu_res", "act3_gelu_grad",
                 "act4_relu_grad", "store_fp32"):
        alpha, bdt, act, rk, _, out_mode, odt, _ = GEMM_PATHS[path]
        A, B, bias, res = gemm_inputs(129, 72, 200, path, seed=3)
        v = alpha * (A.float() @ B.float().t())
        if bias is not None:
            v = v + bias.float()
        z32 = v.clone()
        if act == 1:
            v = v.clamp_min(0)
        elif act == 2:
            v = F.gelu(v)
        elif act == 3:
            a = res.float()
            v = v * (0.5 * (1 + torch.erf(a * 0.7071067811865476)) + a * 0.3989422804014327 * torch.exp(-0.5 * a * a))
        elif act == 4:
            v = torch.where(res.float() > 0, v, torch.zeros_like(v))
        if res is not None and act <= 2:
            v = v + res.float()
        got = v if odt == torch.float32 else v.bfloat16()
        (y, yb), (z, zb) = epilogue_bounds(A, B, alpha, bias, act, res, out_fp32=odt == torch.float32)
        _accept_reject(z32.bfloat16(), z, zb)
        if rk != "cancel":
            _accept_reject(got, y, yb)
            continue
        # the cancellation regime: the product rounded to bf16 before the residual add must be rejected
        _check(got, y, yb, "cpu self-check")
        _must_fail(lambda: _check((z32.bfloat16().float() + res.float()).bfloat16(), y, yb, "perturbed"))


def test_conv_references_match_torch_and_bounds():
    g = torch.Generator().manual_seed(4)
    x = torch.randn(2, 24, 6, 10, generator=g).bfloat16()
    w = (torch.randn(72, 24, 3, 3, generator=g) * 0.1).bfloat16()
    xd = x.double().requires_grad_(True)
    y = F.conv2d(xd, w.double(), None, 2, 1)
    dy = torch.randn(y.shape, generator=g).bfloat16()
    y.backward(dy.double())
    dx64, dxm = conv_dgrad_ref(dy, w, x.shape, 2, 1)
    assert torch.allclose(dx64, xd.grad, rtol=1e-12, atol=1e-12)
    y64, ym = conv_fprop_ref(x, w, 2, 1)
    _accept_reject(F.conv2d(x.float(), w.float(), None, 2, 1).bfloat16(), y64, conv_bound(y64, ym, 9 * 64))
    dx32 = torch.nn.grad.conv2d_input(x.shape, w.float(), dy.float(), 2, 1)
    _accept_reject(dx32.bfloat16(), dx64, conv_bound(dx64, dxm, 9 * 128))


def _bn_fp32(x2, gamma, beta, dz2, eps=BN_EPS):
    """The kernels' formulas evaluated in fp32 on the CPU (one-pass variance)."""
    x = x2.float()
    M = x.shape[0]
    m = x.sum(0) / M
    var = ((x * x).sum(0) / M - m * m).clamp_min(0)
    inv = torch.rsqrt(var + eps)
    g, b = gamma.float(), beta.float()
    a = g * inv
    y = x * a + (b - m * g * inv)
    dz = dz2.float()
    s1, s2 = dz.sum(0), (dz * (x - m)).sum(0)
    xh = (x - m) * inv
    dx = a * (dz - s1 / M - xh * (s2 * inv / M))
    return y, dx, s2 * inv, s1


def test_bn_references_match_torch_and_bounds():
    M, C = 1000, 64
    x2 = bn_inputs(M, C, seed=8)
    g = torch.Generator().manual_seed(9)
    gamma, beta = torch.rand(C, generator=g) + 0.5, 0.3 * torch.randn(C, generator=g)
    dz2 = torch.randn(M, C, generator=g).bfloat16()
    D = standalone_depth(M, C, 132)
    y, yb, _, _ = bn_fwd_bounds(x2, gamma, beta, None, False, D)
    (dx, dxb), (dg, dgb), (db, dbb) = bn_bwd_bounds(x2, dz2, gamma, D, D, False)
    xd = x2.double().requires_grad_(True)
    gd, bd = gamma.double().requires_grad_(True), beta.double().requires_grad_(True)
    yt = F.batch_norm(xd, None, None, gd, bd, True, 0.0, BN_EPS)
    yt.backward(dz2.double())
    assert torch.allclose(y, yt.detach(), rtol=1e-10, atol=1e-10)
    assert torch.allclose(dx, xd.grad, rtol=1e-9, atol=1e-9)
    assert torch.allclose(dg, gd.grad, rtol=1e-9, atol=1e-9)
    assert torch.allclose(db, bd.grad, rtol=1e-9, atol=1e-9)
    y32, dx32, dg32, db32 = _bn_fp32(x2, gamma, beta, dz2)
    _accept_reject(y32.bfloat16(), y, yb)
    _accept_reject(dx32.bfloat16(), dx, dxb)
    _check(dg32, dg, dgb, "cpu self-check")
    _check(db32, db, dbb, "cpu self-check")


def test_pool_references_match_torch_and_bounds():
    x = maxpool_inputs(2, 8, 9, 10, seed=3).bfloat16()
    val, arg = maxpool_ref(x)
    xd = x.double().requires_grad_(True)
    v2, i2 = F.max_pool2d(xd, 3, 2, 1, return_indices=True)
    assert torch.equal(val, v2.detach())
    OH, OW = val.shape[2:]
    kh, kw = arg // 3, arg % 3
    oh = torch.arange(OH).view(1, 1, OH, 1)
    ow = torch.arange(OW).view(1, 1, 1, OW)
    flat = (oh * 2 - 1 + kh) * x.shape[3] + (ow * 2 - 1 + kw)
    assert torch.equal(flat, i2), "reference arg-max is not torch's (first maximum)"
    dy = torch.randn(val.shape, generator=torch.Generator().manual_seed(1)).bfloat16()
    v2.backward(dy.double())
    ref, mag, cnt = maxpool_bwd_ref(dy, arg, x.shape)
    assert torch.allclose(ref, xd.grad, rtol=0, atol=1e-12)
    b = bf16_store(1.01 * (cnt - 1).clamp_min(0) * U32 * mag, ref)
    nz = ref != 0
    _accept_reject(ref.float()[nz].bfloat16(), ref[nz], b[nz])
    xa = torch.randn(3, 16, 7, 7).bfloat16()
    ra = xa.double().mean((2, 3))
    assert torch.allclose(ra, F.adaptive_avg_pool2d(xa.double(), 1).flatten(1), rtol=1e-14, atol=1e-14)
    Ea = 1.01 * 49 * U32 * xa.double().abs().mean((2, 3)) * (1 + 2.02 * U32) + 2.02 * U32 * ra.abs()
    _accept_reject(xa.float().mean((2, 3)).bfloat16(), ra, bf16_store(Ea, ra))
