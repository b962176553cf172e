"""The GEMM epilogues (csrc/gemm_sm90.cu) and the implicit-GEMM convolution forward and data gradient
(csrc/conv_sm90.cu) against float64 on grids where every CTA of ``persistent_body`` (csrc/sm90_common.cuh) walks
many work items.

A CTA carries state from one tile to the next: the operand ring's stage / phase, the epilogue staging tile (and
the residual staged into it), and K loops whose length changes from item to item (the stride-2 data gradient's
parity classes have 1, 2, 2 and 4 taps).  The default grid gives each CTA one tile at the small shapes of
``test_gpu_resnet_numerics.py``, so here every case runs at ``max_ctas`` 1, 3 and 7 (CTAs that walk many items) and
0 (one CTA per SM), with every tile width:
- GEMM: every epilogue path of ``GEMM_PATHS`` at shapes of hundreds of tiles with M / N / K tails, the ResNet-50
  layer-1 1x1 convolution at batch 3 and the ViT-B / GPT-2 linear layers; A and B in both operand layouts for
  the plain, ``bias_f32_alpha_relu_res`` and ``store_fp32`` paths;
- convolution: every convolution of ResNet-50 at 224 x 224 that ``ops.conv.kind`` sends to the implicit-GEMM
  kernel (found by walking the model, not listed by hand), at batch 3, and channel tails (72 / 136 / 200
  channels: several 64-channel chunks per tap, the last one partial).
The first run of a case is checked against float64 with the bounds of ``test_gpu_resnet_numerics.py`` (nothing new
is derived); every other grid and tile width must give the same bits.  Outputs, pre-activations and residuals sit
inside NaN padding (GEMM: ldc padding and guard rows; convolution: guard elements before and after the NHWC
tensor) that must stay NaN, and every launch runs under the host-side launch guard (``launch_guard.py``).

Each case also counts, on the host, the work items the launcher makes and the grid it launches
(``Walk``), and asserts that it is not vacuous (``assert_walks``): at ``max_ctas`` 1 / 3 / 7 some CTA of every
launch runs several items, and 3 or more at some tile width; in the 3x3 stride-2 data gradients some CTA runs items
of different K lengths; the channel-tail cases have at least two channel chunks per tap.
``test_walk_counts_by_hand`` pins that counting on the CPU.
"""
import functools
from dataclasses import dataclass
from typing import List
from unittest import mock

import pytest
import torch

import launch_guard
from fp64_bounds import assert_within_bound, report_ratios
from test_gpu_resnet_numerics import (GEMM_PATHS, _check_split, _choose_box, _pad64, conv_bound, conv_dgrad_ref,
                                      conv_fprop_ref, epilogue_bounds, gemm_inputs)

gpu = pytest.mark.gpu

MAX_CTAS = (1, 3, 7, 0)
GEMM_BLOCK_NS = (0, 64, 128, 256)
CONV_BLOCK_NS = (64, 128)
GUARD_ROWS = 3             # NaN rows above and below every GEMM output, pre-activation and residual
GUARD = 72                 # NaN elements before and after every convolution output (a multiple of 8: 16-byte base)
STATS_MAX_CTAS = 256       # sm90_common.cuh: launch_persistent never launches more CTAs than that


@pytest.fixture(scope="module", autouse=True)
def _report_ratios():
    yield
    report_ratios()


@pytest.fixture
def guard(monkeypatch):
    from distributed_torch_horovod_gcp_b200.ops import kernels
    assert kernels.has("gemm") and kernels.has("conv_implicit_gemm"), "libb200dp_kernels.so not loaded"
    return launch_guard.install(monkeypatch)


# ================================================================================================ work-item count
def _cdiv(a, b):
    return -(-a // b)


def pick_bn(n, block_n):
    """sm90_common.cuh ``pick_bn``: the tile width a launch runs (0: by the output width; 256 runs as 128)."""
    if block_n == 0:
        return 128 if n > 64 else 64
    return min(block_n, 128)


@dataclass
class Walk:
    """The work items of one persistent launch (their 64-deep K-block counts, in item order) and its grid:
    ``launch_persistent`` launches min(items, SMs, max_ctas if > 0, 256) CTAs and CTA b runs items b, b + grid, ..."""
    kbs: List[int]
    grid: int

    @classmethod
    def of(cls, kbs, sms, max_ctas):
        grid = min(len(kbs), sms, STATS_MAX_CTAS)
        if max_ctas > 0:
            grid = min(grid, max_ctas)
        return cls(kbs, grid)

    def cta(self, b):
        return self.kbs[b::self.grid]

    @property
    def most(self):
        """Items of the busiest CTA."""
        return max(len(self.cta(b)) for b in range(self.grid))

    @property
    def mixed_k(self):
        """Whether some CTA runs items of different K lengths."""
        return any(len(set(self.cta(b))) > 1 for b in range(self.grid))


def gemm_walk(M, N, K, block_n, max_ctas, sms):
    """gemm_sm90.cu without split-K: one item per 128 x BN output tile, ceil(K / 64) K blocks each."""
    items = _cdiv(M, 128) * _cdiv(N, pick_bn(N, block_n))
    return Walk.of([_cdiv(K, 64)] * items, sms, max_ctas)


def conv_class_taps(mode, R, stride):
    """Taps of each class of conv_sm90.cu: fprop and stride-1 dgrad one class of R*R taps; stride-2 dgrad one
    class per parity (ph, pw) of dx, in that order, with the taps (r, s) of matching parity, empty classes dropped."""
    if mode == "fprop" or stride == 1:
        return [R * R]
    pad = (R - 1) // 2
    taps = []
    for ph in (0, 1):
        for pw in (0, 1):
            n = sum(1 for r in range(R) if (ph + pad - r) % 2 == 0) * \
                sum(1 for s in range(R) if (pw + pad - s) % 2 == 0)
            if n:
                taps.append(n)
    return taps


def kc_per_tap(mode, Cin, Cout):
    """64-channel chunks of the reduction per tap: Cin for fprop, Cout for dgrad."""
    return _cdiv(Cin if mode == "fprop" else Cout, 64)


def conv_walk(mode, N, Cin, H, W, Cout, R, stride, block_n, max_ctas, sms):
    """conv_sm90.cu fprop / dgrad: items = class x pixel tile x n block (n fastest), pixel tiles = the
    ``choose_box`` boxes of 128 output pixels over (OW, OH, N) (for dgrad at stride 2: one parity view of dx),
    K blocks = the class's taps x ``kc_per_tap``."""
    OH, OW = H // stride, W // stride
    bw, bh, bn = _choose_box(OW, OH, N, 128)
    pix = _cdiv(OW, bw) * _cdiv(OH, bh) * _cdiv(N, bn)
    n_out = Cout if mode == "fprop" else Cin
    nnb = _cdiv(n_out, pick_bn(n_out, block_n))
    kc = kc_per_tap(mode, Cin, Cout)
    return Walk.of([t * kc for t in conv_class_taps(mode, R, stride) for _ in range(pix * nnb)], sms, max_ctas)


def assert_walks(walks, mixed=False):
    """``walks``: {(block_n, max_ctas): Walk} of one operation of a case.  At max_ctas 1 / 3 / 7 every launch has
    a CTA that runs more than one item, and at least one tile width has a CTA that runs 3 or more (the widest
    tiles of the 7 x 7 ResNet-50 layers at batch 3 make too few items for 3 on each of 7 CTAs); with ``mixed``
    (the 3x3 stride-2 data gradient) every such launch has a CTA that runs items of different K lengths."""
    for mc in (1, 3, 7):
        at = {bn: w for (bn, m), w in walks.items() if m == mc}
        for bn, w in at.items():
            assert w.most >= 2, f"block_n={bn} max_ctas={mc}: every CTA runs one item ({len(w.kbs)} items)"
            assert not mixed or w.mixed_k, f"block_n={bn} max_ctas={mc}: no CTA runs items of different K lengths"
        assert max(w.most for w in at.values()) >= 3, f"max_ctas={mc}: no CTA runs 3 items at any tile width"


def test_walk_counts_by_hand():
    """Two launches counted by hand on a 132-SM H100.
    GEMM 1000 x 264 x 200, BN 64: 8 m blocks x 5 n blocks = 40 tiles of 4 K blocks; at max_ctas 7, CTA 0 runs
    tiles 0, 7, .., 35 (6) and CTA 6 runs 6, 13, .., 34 (5); on the default grid each of 40 CTAs runs one.
    dgrad 3x3 stride 2 of x [3, 128, 56, 56] (dy 28 x 28), Cout 128, BN 64: the 128-pixel box of 28 x 28 x 3 with
    the least padding is 32 x 4 x 1 (28 x 32 x 3 and 32 x 28 x 3 both cover 2688 pixels; the wider wins), so
    1 x 7 x 3 = 21 pixel tiles; parity classes of 1, 2, 2, 4 taps x 2 channel chunks = 2, 4, 4, 8 K blocks;
    2 n blocks: 4 x 21 x 2 = 168 items.  On 132 CTAs, CTA 0 runs item 0 (class 0: 2 K blocks) and item 132
    (class 132 // 42 = 3: 8 K blocks); CTA 36 runs item 36 alone."""
    w = gemm_walk(1000, 264, 200, 64, 7, 132)
    assert (len(w.kbs), set(w.kbs), w.grid) == (40, {4}, 7)
    assert w.cta(0) == [4] * 6 and w.cta(6) == [4] * 5 and w.most == 6
    w = gemm_walk(1000, 264, 200, 64, 0, 132)
    assert (w.grid, w.most) == (40, 1)
    assert gemm_walk(1000, 264, 200, 256, 0, 132).kbs == gemm_walk(1000, 264, 200, 128, 0, 132).kbs == [4] * 24

    assert _choose_box(28, 28, 3, 128) == (32, 4, 1)
    assert conv_class_taps("dgrad", 3, 2) == [1, 2, 2, 4]
    assert conv_class_taps("dgrad", 1, 2) == [1]
    w = conv_walk("dgrad", 3, 128, 56, 56, 128, 3, 2, 64, 0, 132)
    assert (len(w.kbs), w.grid) == (168, 132)
    assert w.kbs == [2] * 42 + [4] * 84 + [8] * 42
    assert w.cta(0) == [2, 8] and w.cta(36) == [2] and w.mixed_k and w.most == 2
    w = conv_walk("dgrad", 3, 128, 56, 56, 128, 3, 2, 64, 1, 132)
    assert w.grid == 1 and w.most == 168 and w.mixed_k


# ================================================================================================ ResNet-50 walk
class _ReportsCuda(torch.Tensor):
    """A CPU activation that ``ops.conv.kind`` takes for a CUDA one (the walk needs no GPU)."""

    @property
    def is_cuda(self):
        return True


@functools.lru_cache(maxsize=None)
def resnet50_implicit_convs(batch=3, size=224):
    """(N, Cin, H, W, Cout, R, stride) of every distinct convolution of ``models.resnet50()`` at size x size that
    ``ops.conv.kind`` sends to ``"implicit"``.  The model's forward runs once on the CPU with every
    conv + BN (+ ReLU) unit of the functional layer replaced by a recorder, which notes the convolution and its
    input and returns zeros of the output's shape; then ``kind`` judges each one with the kernel library taken as
    loaded."""
    from distributed_torch_horovod_gcp_b200 import models
    from distributed_torch_horovod_gcp_b200.ops import bn, conv, functional, gemm
    seen = []

    def record(x, cv, bnm, relu=True, residual=None):
        seen.append((cv, tuple(x.shape)))
        N, _, H, W = x.shape
        (R, S), (sh, sw), (ph, pw) = cv.kernel_size, cv.stride, cv.padding
        return x.new_zeros(N, cv.out_channels, (H + 2 * ph - R) // sh + 1, (W + 2 * pw - S) // sw + 1)

    model = models.resnet50()
    with mock.patch.object(functional, "conv_bn_act", record), torch.no_grad():
        model(torch.zeros(batch, 3, size, size))
    loaded = type("Loaded", (), {"b200dp_stem_im2col": None})()
    cases = []
    with mock.patch.object(bn, "_lib", loaded), mock.patch.object(gemm, "_lib", loaded), \
            mock.patch.object(conv, "_lib", loaded):
        for cv, (N, C, H, W) in seen:
            x = torch.empty(N, C, H, W, dtype=torch.bfloat16, memory_format=torch.channels_last)
            if conv.kind(x.as_subclass(_ReportsCuda), cv.to(torch.bfloat16)) == "implicit":
                case = (N, C, H, W, cv.out_channels, cv.kernel_size[0], cv.stride[0])
                if case not in cases:
                    cases.append(case)
    return cases


def test_resnet50_walk_finds_the_implicit_convolutions():
    """The walk sees the 3x3 convolutions at stride 1 on 56 / 28 / 14 / 7 and stride 2 from 56 / 28 / 14, and the
    strided 1x1 downsamples; never the stem or a 1x1 stride-1 convolution (the GEMM takes those)."""
    cases = resnet50_implicit_convs()
    got = {(R, s, H) for _, _, H, _, _, R, s in cases}
    assert {(3, 1, h) for h in (56, 28, 14, 7)} | {(3, 2, h) for h in (56, 28, 14)} | \
        {(1, 2, h) for h in (56, 28, 14)} == got
    assert len(cases) == 10 and all(c[0] == 3 and c[2] == c[3] for c in cases)


# N, Cin, H, W, Cout, R, stride: channel tails on both sides (fprop reduces Cin, dgrad reduces Cout)
TAIL_CASES = [
    (3, 72, 28, 28, 200, 3, 1),
    (3, 136, 56, 56, 72, 3, 2),
    (3, 200, 28, 28, 136, 3, 2),
    (3, 72, 56, 56, 136, 1, 2),
    (3, 200, 56, 56, 72, 1, 2),
]


def _conv_id(c):
    N, Cin, H, W, Cout, R, s = c
    return f"{R}x{R}s{s}-{N}x{Cin}x{H}x{W}-{Cout}"


# ================================================================================================ GEMM
# M, N, K, extra (ldc - N)
WALK_GEMM_SHAPES = [(1000, 264, 200, 8), (4099, 776, 72, 24), (9408, 256, 64, 16),
                    (788, 2304, 768, 8), (788, 768, 3072, 16), (8192, 768, 768, 8)]
LAYOUT_PATHS = ("plain", "bias_f32_alpha_relu_res", "store_fp32")
LAYOUTS = [(False, False), (False, True), (True, False), (True, True)]     # (a_mn, b_mn)


def _default_layout(path):
    """As ``run_gemm_path``: the residual / aux paths are dgrad GEMMs (B MN-major), the others forward GEMMs."""
    return (False, GEMM_PATHS[path][3] is not None)


def _layout_id(lay):
    return f"A{'mn' if lay[0] else 'k'}-B{'mn' if lay[1] else 'k'}"


GEMM_CASES = [(p, lay) for p in GEMM_PATHS if p != "res_mask"
              for lay in (LAYOUTS if p in LAYOUT_PATHS else [_default_layout(p)])]


def _nan_rows(rows, ld, dtype):
    """A [GUARD_ROWS + rows + GUARD_ROWS, ld] NaN buffer and its [rows, ld] body."""
    big = torch.full((rows + 2 * GUARD_ROWS, ld), float("nan"), dtype=dtype, device="cuda")
    return big, big[GUARD_ROWS:GUARD_ROWS + rows]


def _only_nan_outside(big, rows, cols, what):
    body = torch.zeros_like(big, dtype=torch.bool)
    body[GUARD_ROWS:GUARD_ROWS + rows, :cols] = True
    assert bool(big[~body].isnan().all()), f"{what} written outside its [{rows}, {cols}] body"


def _operand(X, mn):
    """X [rows, K] stored K-major ([rows][K + 8]) or MN-major ([K][rows rounded up to 8, + 8]), the padding NaN,
    as the [rows, K] / [K, rows] view the kernel reads."""
    rows, K = X.shape
    if mn:
        buf = torch.full((K, 8 * _cdiv(rows, 8) + 8), float("nan"), dtype=X.dtype, device="cuda")
        buf[:, :rows] = X.t().cuda()
        return buf[:, :rows]
    buf = torch.full((rows, K + 8), float("nan"), dtype=X.dtype, device="cuda")
    buf[:, :K] = X.cuda()
    return buf[:, :K]


def _bits(t):
    return t.view(torch.int16 if t.element_size() == 2 else torch.int32)


def run_walking_gemm(path, M, N, K, extra, a_mn, b_mn):
    from distributed_torch_horovod_gcp_b200.ops import gemm as gm
    alpha, bdt, act, rk, want_pre, out_mode, odt, use_mask = GEMM_PATHS[path]
    A, B, bias, res = gemm_inputs(M, N, K, path, seed=7 * M + 3 * N + K)
    ldc = N + extra
    a, b = _operand(A, a_mn), _operand(B, b_mn)
    bias_d = bias.cuda() if bias is not None else None
    bits, res_used = None, res
    if use_mask:
        gk = torch.Generator().manual_seed(7 * M + 3 * N + K + 1)
        keep = torch.rand(M, N, generator=gk) > 0.4
        bits = (keep.view(M, N // 8, 8).to(torch.uint8) << torch.arange(8, dtype=torch.uint8)).sum(2)
        bits = bits.to(torch.uint8).contiguous().cuda()
        res_used = res * keep.bfloat16()
    res_big = res_body = None
    if res is not None:
        res_big, res_body = _nan_rows(M, ldc, torch.bfloat16)
        res_body[:, :N] = res.cuda()
        res_before = res_big.clone()
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    assert_walks({(bn, mc): gemm_walk(M, N, K, bn, mc, sms) for bn in GEMM_BLOCK_NS for mc in MAX_CTAS})
    first = ref = None
    for bn in GEMM_BLOCK_NS:
        for mc in MAX_CTAS:
            out_big, out = _nan_rows(M, ldc, odt)
            pre_big, pre = _nan_rows(M, ldc, torch.bfloat16) if want_pre else (None, None)
            gm.gemm(a, b, out[:, :N], M, N, K, a_mn=a_mn, b_mn=b_mn, bias=bias_d,
                    residual=res_body[:, :N] if res is not None else None,
                    preact=pre[:, :N] if want_pre else None, act=act, out_mode=out_mode, alpha=alpha,
                    block_n=bn, max_ctas=mc, res_mask=bits)
            torch.cuda.synchronize()
            tag = f"block_n={bn} max_ctas={mc}"
            _only_nan_outside(out_big, M, N, f"output ({tag})")
            if want_pre:
                _only_nan_outside(pre_big, M, N, f"preact ({tag})")
            if res is not None:
                assert torch.equal(_bits(res_big), _bits(res_before)), f"residual buffer changed ({tag})"
            if first is None:
                (y, yb), (z, zb) = epilogue_bounds(A.cuda(), B.cuda(), alpha, bias_d, act,
                                                   res_used.cuda() if res_used is not None else None,
                                                   out_fp32=odt == torch.float32)
                assert_within_bound(out[:, :N], y, group=f"walking gemm {path}", terms=[(1.0, yb)])
                if want_pre:
                    assert_within_bound(pre[:, :N], z, group="walking gemm preact", terms=[(1.0, zb)])
                first = (out_big, pre_big)
                ref = tag
            else:
                assert torch.equal(_bits(out_big), _bits(first[0])), f"output: {tag} differs from {ref}"
                if want_pre:
                    assert torch.equal(_bits(pre_big), _bits(first[1])), f"preact: {tag} differs from {ref}"


@gpu
@pytest.mark.parametrize("shape", WALK_GEMM_SHAPES, ids=lambda s: "x".join(map(str, s[:3])))
@pytest.mark.parametrize("path,layout", GEMM_CASES, ids=[f"{p}-{_layout_id(lay)}" for p, lay in GEMM_CASES])
def test_walking_gemm_epilogue_vs_fp64(path, layout, shape, guard):
    M, N, K, extra = shape
    run_walking_gemm(path, M, N, K, extra, *layout)
    assert guard["b200dp_gemm_bf16"] == len(GEMM_BLOCK_NS) * len(MAX_CTAS)


@gpu
@pytest.mark.parametrize("shape", [s for s in WALK_GEMM_SHAPES if s[1] % 64 == 0],
                         ids=lambda s: "x".join(map(str, s[:3])))
def test_walking_gemm_res_mask_vs_fp64(shape, guard):
    """The ReLU-mask residual takes dense rows (ldc = N) and N % 64 == 0: no ldc padding, only guard rows."""
    M, N, K, _ = shape
    run_walking_gemm("res_mask", M, N, K, 0, *_default_layout("res_mask"))
    assert guard["b200dp_gemm_bf16"] == len(GEMM_BLOCK_NS) * len(MAX_CTAS)


# ================================================================================================ convolution
def _guarded_nhwc(N, C, H, W):
    """A NaN buffer of GUARD + N*H*W*C + GUARD bf16 elements and the [N, C, H, W] channels_last view of its body."""
    n = N * C * H * W
    buf = torch.full((n + 2 * GUARD,), float("nan"), dtype=torch.bfloat16, device="cuda")
    return buf, buf[GUARD:GUARD + n].view(N, H, W, C).permute(0, 3, 1, 2)


def _guards_nan(buf):
    return bool(buf[:GUARD].isnan().all()) and bool(buf[-GUARD:].isnan().all())


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _check_dgrad_parities(dx, dx64, dxb, R):
    """Stride 2: each parity class of dx on its own; with a 1x1 filter the odd rows / columns get no tap and are
    exact zeros."""
    for ph in (0, 1):
        for pw in (0, 1):
            sl = (slice(None), slice(None), slice(ph, None, 2), slice(pw, None, 2))
            if R == 1 and (ph or pw):
                assert float(dx64[sl].abs().max()) == 0.0
                assert bool((dx[sl] == 0).all()), f"1x1 s2 dgrad: parity ({ph}, {pw}) not zero"
            else:
                assert float(dx64[sl].abs().max()) > 0.0
                assert_within_bound(dx[sl], dx64[sl], group="walking conv dgrad s2 parity classes",
                                    terms=[(1.0, dxb[sl])])


def run_walking_conv(N, Cin, H, W, Cout, R, stride, tails=False):
    from distributed_torch_horovod_gcp_b200.ops import conv
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    pad = (R - 1) // 2
    OH, OW = H // stride, W // stride
    g = torch.Generator(device="cuda").manual_seed(N * H * W + 5 * Cin + 3 * Cout + 11 * R + stride)
    x = torch.randn(N, Cin, H, W, device="cuda", generator=g).bfloat16().contiguous(memory_format=torch.channels_last)
    w = (torch.randn(Cout, Cin, R, R, device="cuda", generator=g) * (Cin * R * R) ** -0.5).bfloat16() \
        .contiguous(memory_format=torch.channels_last)
    dy = torch.randn(N, Cout, OH, OW, device="cuda", generator=g).bfloat16() \
        .contiguous(memory_format=torch.channels_last)
    y64, ym = conv_fprop_ref(x, w, stride, pad)
    yb = conv_bound(y64, ym, R * R * _pad64(Cin))
    dx64, dxm = conv_dgrad_ref(dy, w, x.shape, stride, pad)
    dxb = conv_bound(dx64, dxm, R * R * _pad64(Cout))
    for mode in ("fprop", "dgrad"):
        assert_walks({(bn, mc): conv_walk(mode, N, Cin, H, W, Cout, R, stride, bn, mc, sms)
                      for bn in CONV_BLOCK_NS for mc in MAX_CTAS}, mixed=mode == "dgrad" and stride == 2 and R == 3)
        assert not tails or kc_per_tap(mode, Cin, Cout) >= 2, f"{mode}: one channel chunk per tap"
    first = None
    for bn in CONV_BLOCK_NS:
        for mc in MAX_CTAS:
            tag = f"block_n={bn} max_ctas={mc}"
            ybuf, y = _guarded_nhwc(N, Cout, OH, OW)
            rc = conv._lib.b200dp_conv_fprop(x.data_ptr(), w.data_ptr(), y.data_ptr(), N, H, W, Cin, Cout, R, R,
                                             stride, pad, bn, mc, None, _stream())
            assert rc == 0, conv._lib.b200dp_conv_last_error()
            dxbuf, dx = _guarded_nhwc(N, Cin, H, W)
            rc = conv._lib.b200dp_conv_dgrad(dy.data_ptr(), w.data_ptr(), dx.data_ptr(), N, H, W, Cin, Cout, R, R,
                                             stride, pad, bn, mc, _stream())
            assert rc == 0, conv._lib.b200dp_conv_last_error()
            torch.cuda.synchronize()
            assert _guards_nan(ybuf), f"fprop wrote outside its output ({tag})"
            assert _guards_nan(dxbuf), f"dgrad wrote outside its output ({tag})"
            if first is None:
                _check_split(y, y64, yb, "walking conv fprop")
                _check_split(dx, dx64, dxb, "walking conv dgrad")
                if stride == 2:
                    _check_dgrad_parities(dx, dx64, dxb, R)
                first, ref = (ybuf, dxbuf), tag
            else:
                assert torch.equal(_bits(ybuf), _bits(first[0])), f"fprop: {tag} differs from {ref}"
                assert torch.equal(_bits(dxbuf), _bits(first[1])), f"dgrad: {tag} differs from {ref}"


@gpu
@pytest.mark.parametrize("case", resnet50_implicit_convs(), ids=_conv_id)
def test_walking_conv_resnet50_vs_fp64(case, guard):
    from distributed_torch_horovod_gcp_b200.ops import conv
    N, Cin, H, W, Cout, R, stride = case
    x = torch.empty(N, Cin, H, W, device="cuda", dtype=torch.bfloat16, memory_format=torch.channels_last)
    cv = torch.nn.Conv2d(Cin, Cout, R, stride, (R - 1) // 2, bias=False).cuda().bfloat16()
    assert conv.kind(x, cv) == "implicit"
    run_walking_conv(*case)
    n = len(CONV_BLOCK_NS) * len(MAX_CTAS)
    assert guard["b200dp_conv_fprop"] == n and guard["b200dp_conv_dgrad"] == n


@gpu
@pytest.mark.parametrize("case", TAIL_CASES, ids=_conv_id)
def test_walking_conv_channel_tails_vs_fp64(case, guard):
    run_walking_conv(*case, tails=True)
    n = len(CONV_BLOCK_NS) * len(MAX_CTAS)
    assert guard["b200dp_conv_fprop"] == n and guard["b200dp_conv_dgrad"] == n
