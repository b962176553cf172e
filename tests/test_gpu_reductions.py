"""Fixed-order cross-CTA reductions, checked bit for bit and against float64.

Every cross-CTA reduction on the ResNet training path sums its parts in a fixed order, so a training
step computes the same bits on every run:

- split-K GEMM / convolution weight gradient (``splitk_finish_tile``): each split stores its partial tile
  into its own fp32 workspace slice; the last split to arrive sums the slices in split order and adds the
  sum to C, or stores it, in C's dtype;
- BatchNorm statistics from the GEMM / convolution epilogue (``stats_flush`` / ``stats_finalize``) and the
  stand-alone BatchNorm reductions (``block_reduce_to_global``): every CTA writes its own slot and the last
  CTA sums the slots in CTA order.

The tests below check that order exactly (a split-K result must equal the per-split partials of the same
kernel summed in split order, for any grid size), that results are independent of the grid, that the add /
store modes write in bf16 or fp32 exactly the bits of adding into a zeroed fp32 buffer and converting that,
that fp32 outputs lie within a rigorous per-element bound of a float64 reference of the same operation, and
that a whole ResNet training step repeats bit for bit.

Not covered on purpose: ViT and LSTM training are not reproducible run to run.  The LayerNorm parameter
gradients (``elementwise.cu``), the attention dQ accumulation (``attn_sm90.cu``) and the LSTM ``dW_hh``
(``lstm_rec_sm90.cu``) still sum with fp32 atomics, in arrival order.
"""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
U32 = 2.0 ** -24          # unit roundoff of fp32
U_BF16 = 2.0 ** -8        # relative rounding error of a bf16 store

# worst err/bound ratio seen per test group (printed at the end of the module, e.g. with `pytest -s`)
_WORST = {}


@pytest.fixture(scope="module", autouse=True)
def _report_ratios():
    yield
    for k in sorted(_WORST):
        print(f"\n[err/bound] {k}: max {_WORST[k]:.3e}", end="")
    print()


def _assert_within_bound(out, ref64, mag64, n_terms, out_bf16=False, group="misc"):
    """|out - ref64| <= 2 * n_terms * 2^-24 * mag64 (+ 2^-8 * |ref64| for a bf16 output), elementwise.

    ``ref64``: the operation in float64 on the bf16 inputs the kernel saw; ``mag64``: the same operation on
    absolute values.  This bounds any fp32 summation order and rounding of ``n_terms`` terms, so it needs no
    fitting and does not flake."""
    out64 = out.double()
    err = (out64 - ref64).abs()
    bound = 2.0 * n_terms * U32 * mag64
    if out_bf16:
        bound = bound + U_BF16 * ref64.abs()
    ratio = torch.where(bound > 0, err / bound.clamp_min(1e-300),
                        torch.where(err > 0, torch.full_like(err, float("inf")), torch.zeros_like(err)))
    worst = int(torch.argmax(ratio))
    r = float(ratio.reshape(-1)[worst])
    _WORST[group] = max(_WORST.get(group, 0.0), r)
    if not bool((err <= bound).all()):
        idx = np.unravel_index(worst, tuple(ratio.shape))
        raise AssertionError(
            f"{group}: {int((err > bound).sum())} element(s) outside the fp64 bound; worst at {tuple(map(int, idx))}: "
            f"out={float(out64[idx]):.9g} ref={float(ref64[idx]):.9g} err/bound={r:.3g}")


def _gemm():
    from distributed_torch_horovod_gcp_b200.ops import gemm, kernels
    assert kernels.has("gemm"), "libb200dp_kernels.so not loaded / gemm symbol missing"
    return gemm


def _conv_lib():
    from distributed_torch_horovod_gcp_b200.ops import conv, kernels
    assert kernels.has("conv_implicit_gemm"), "conv kernel missing from libb200dp_kernels.so"
    return conv._lib


def _bn_lib():
    from distributed_torch_horovod_gcp_b200.ops import bn, kernels
    assert kernels.has("bn_act"), "BatchNorm kernels missing from libb200dp_kernels.so"
    return bn._lib


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _cdiv(a, b):
    return -(-a // b)


# ------------------------------------------------------------------------------------------------ GEMM split-K

def _operands(M, N, K, a_mn, b_mn, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    A = torch.randn(M, K, device="cuda", generator=g).to(torch.bfloat16)
    B = torch.randn(N, K, device="cuda", generator=g).to(torch.bfloat16)
    a = A.t().contiguous() if a_mn else A
    b = B.t().contiguous() if b_mn else B
    return A, B, a, b


def _splitk_expected(g, a, b, C0, M, N, K, a_mn, b_mn, alpha, splits, block_n):
    """The split-K result rebuilt from its parts: the same kernel, unsplit, on each split's K range
    (host normalisation of ``splits`` replicated), the partials summed in split order in fp32, then added
    to the prior contents ``C0``."""
    kb = _cdiv(K, 64)
    s = min(splits, kb)
    per = _cdiv(kb, s)
    s = _cdiv(kb, per)
    acc = None
    for k in range(s):
        k0, k1 = k * per * 64, min((k + 1) * per * 64, K)
        ak = a[k0:k1] if a_mn else a[:, k0:k1]
        bk = b[k0:k1] if b_mn else b[:, k0:k1]
        p = torch.empty(M, N, device="cuda", dtype=torch.float32)
        g.gemm(ak, bk, p, M, N, k1 - k0, a_mn=a_mn, b_mn=b_mn, out_mode=2, alpha=alpha, block_n=block_n)
        acc = p if acc is None else acc + p
    return C0 + acc, s


SPLITK_CASES = [
    # a_mn, b_mn, M, N, K, block_n, splits, alpha, extra ldc columns
    (False, False, 1000, 200, 576, 128, 4, 1.0, 0),      # kb = 9: 4 splits normalise to 3
    (False, True, 1000, 264, 200, 64, 3, 1.0, 0),        # K tail block; 3 -> 2 splits
    (True, False, 1000, 200, 1024, 128, 5, 0.5, 24),     # alpha, out is a column slice (ldc > N)
    (True, True, 1000, 264, 72, 64, 7, 1.0, 0),          # more splits than K blocks
    (True, True, 1000, 264, 640, 128, 10, -1.25, 8),     # one K block per split
    (False, False, 1000, 200, 200, 64, 4, 2.0, 0),
    (False, True, 1000, 264, 1000, 128, 6, 1.0, 0),
    (True, False, 1000, 200, 456, 64, 2, 1.0, 16),
]


@pytest.mark.parametrize("a_mn,b_mn,M,N,K,block_n,splits,alpha,extra", SPLITK_CASES)
def test_gemm_splitk_sums_in_split_order(a_mn, b_mn, M, N, K, block_n, splits, alpha, extra):
    g = _gemm()
    A, B, a, b = _operands(M, N, K, a_mn, b_mn, seed=K + N)
    ldc = N + extra
    big0 = torch.randn(M, ldc, device="cuda", dtype=torch.float32)
    C0 = big0[:, :N].clone()
    expected, s = _splitk_expected(g, a, b, C0, M, N, K, a_mn, b_mn, alpha, splits, block_n)
    ref64 = C0.double() + alpha * (A.double() @ B.double().t())
    mag64 = C0.double().abs() + abs(alpha) * (A.double().abs() @ B.double().abs().t())
    for max_ctas in (0, 1, 3, 7):
        big = big0.clone()
        out = big[:, :N]
        g.gemm(a, b, out, M, N, K, a_mn=a_mn, b_mn=b_mn, out_mode=1, splits=splits, alpha=alpha,
               block_n=block_n, max_ctas=max_ctas)
        torch.cuda.synchronize()
        assert torch.equal(out, expected), \
            f"max_ctas={max_ctas}: split-K != partials summed in split order " \
            f"(max diff {float((out - expected).abs().max()):.3g})"
        if extra:
            assert torch.equal(big[:, N:], big0[:, N:]), "split-K wrote past column N of its output"
        _assert_within_bound(out, ref64, mag64, K + s + 1, group="gemm split-K")


def test_gemm_bias_grad_shape_splitk():
    """ops.gemm.bias_grad: column sums of dz as a GEMM against a ones [M, 8] MN-major operand, N = 8,
    64-wide tiles, many splits over a long K."""
    g = _gemm()
    C, rows = 256, 8 * 56 * 56
    gen = torch.Generator(device="cuda").manual_seed(7)
    dz = torch.randn(rows, C, device="cuda", generator=gen).to(torch.bfloat16)     # [K, M]: MN-major A
    ones = torch.ones(rows, 8, device="cuda", dtype=torch.bfloat16)                # [K, N]: MN-major B
    kb = _cdiv(rows, 64)
    splits = max(1, min(kb // 4, (2 * 132) // _cdiv(C, 128)))
    C0 = torch.zeros(C, 8, device="cuda", dtype=torch.float32)
    expected, s = _splitk_expected(g, dz, ones, C0, C, 8, rows, True, True, 1.0, splits, 64)
    assert s > 64
    ref64 = dz.double().sum(0)[:, None].expand(C, 8)
    mag64 = dz.double().abs().sum(0)[:, None].expand(C, 8)
    for max_ctas in (0, 1, 3, 7):
        out = torch.zeros(C, 8, device="cuda", dtype=torch.float32)
        g.gemm(dz, ones, out, C, 8, rows, a_mn=True, b_mn=True, out_mode=1, splits=splits, block_n=64,
               max_ctas=max_ctas)
        torch.cuda.synchronize()
        assert torch.equal(out, expected), f"max_ctas={max_ctas}"
        _assert_within_bound(out, ref64, mag64, rows + s + 1, group="gemm split-K")
    db = g.bias_grad(dz, C, rows, torch.float32)
    assert torch.equal(db, expected[:, 0])


def test_gemm_splitk_on_side_streams():
    """Split-K takes its workspace per launch on the launch stream: two different split-K GEMMs issued
    alternately on two streams, without synchronisation in between, each give their single-stream bits."""
    g = _gemm()
    cfgs = [(False, True, 1000, 264, 640, 128, 4), (True, True, 512, 200, 1024, 64, 6)]
    ops, ref = [], []
    for i, (a_mn, b_mn, M, N, K, bn, s) in enumerate(cfgs):
        _, _, a, b = _operands(M, N, K, a_mn, b_mn, seed=100 + i)
        C0 = torch.randn(M, N, device="cuda", dtype=torch.float32)
        out = C0.clone()
        g.gemm(a, b, out, M, N, K, a_mn=a_mn, b_mn=b_mn, out_mode=1, splits=s, block_n=bn)
        ops.append((a, b, C0, M, N, K, a_mn, b_mn, s, bn))
        ref.append(out)
    reps = 4
    outs = [[op[2].clone() for _ in range(reps)] for op in ops]
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    main = torch.cuda.current_stream()
    for st in streams:
        st.wait_stream(main)
    for r in range(reps):
        for i, (a, b, C0, M, N, K, a_mn, b_mn, s, bn) in enumerate(ops):
            with torch.cuda.stream(streams[(i + r) % 2]):
                g.gemm(a, b, outs[i][r], M, N, K, a_mn=a_mn, b_mn=b_mn, out_mode=1, splits=s, block_n=bn)
    for st in streams:
        main.wait_stream(st)
    torch.cuda.synchronize()
    for i in range(len(ops)):
        for r in range(reps):
            assert torch.equal(outs[i][r], ref[i]), (i, r)


# ------------------------------------------------------------------------------------------------ add / store modes

def _assert_same_bits(out, ref, what):
    """Bit patterns, not values: torch.equal treats -0.0 == +0.0."""
    itype = torch.int16 if out.dtype == torch.bfloat16 else torch.int32
    diff = out.contiguous().view(itype) != ref.contiguous().view(itype)
    if bool(diff.any()):
        i = int(diff.reshape(-1).nonzero()[0])
        raise AssertionError(f"{what}: {int(diff.sum())} element(s) differ from the two-stage bits, first: "
                             f"out={float(out.reshape(-1)[i])!r} ref={float(ref.reshape(-1)[i])!r}")


def _two_stage(add_into_zeros, prior, acc):
    """What the add (``acc``) / store modes must write: the same kernel adds into a zeroed fp32 buffer, and
    (prior + buffer), or the buffer alone, is rounded once to the prior's dtype.  A -0 sum thus comes out +0."""
    buf = torch.zeros(prior.shape, device="cuda", dtype=torch.float32)
    add_into_zeros(buf)
    return ((prior.float() + buf) if acc else buf).to(prior.dtype)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
@pytest.mark.parametrize("a_mn,b_mn,M,N,K,block_n,splits,alpha,extra", SPLITK_CASES)
def test_gemm_add_store_match_two_stage_bits(a_mn, b_mn, M, N, K, block_n, splits, alpha, extra, dtype):
    """out_mode 1 (add) and 2 (store) into a bf16 or fp32 C, split-K and one split, for every grid cap.
    Rows 0..7 of A are zero against an all-negative B, so whole rows of the product are signed zeros, and
    the prior contents there are -0."""
    g = _gemm()
    A, B, a, b = _operands(M, N, K, a_mn, b_mn, seed=K + N + 1)
    B.abs_().neg_()
    A[:8] = 0
    a = A.t().contiguous() if a_mn else A
    b = B.t().contiguous() if b_mn else B
    ldc = N + extra
    prior_big = torch.randn(M, ldc, device="cuda").to(dtype)
    prior_big[:8] = -0.0
    prior = prior_big[:, :N]
    for s in (splits, 1):
        def add_into_zeros(buf):
            g.gemm(a, b, buf, M, N, K, a_mn=a_mn, b_mn=b_mn, out_mode=1, splits=s, alpha=alpha, block_n=block_n)
        for acc in (False, True):
            ref = _two_stage(add_into_zeros, prior, acc)
            for max_ctas in (0, 1, 3, 7):
                big = prior_big.clone() if acc else torch.full_like(prior_big, float("nan"))
                g.gemm(a, b, big[:, :N], M, N, K, a_mn=a_mn, b_mn=b_mn, out_mode=1 if acc else 2, splits=s,
                       alpha=alpha, block_n=block_n, max_ctas=max_ctas)
                torch.cuda.synchronize()
                _assert_same_bits(big[:, :N], ref, f"splits={s} acc={acc} max_ctas={max_ctas}")
                if extra:
                    _assert_same_bits(big[:, N:], prior_big[:, N:] if acc else torch.full_like(big[:, N:], float("nan")),
                                      "columns past N")
    # the crafted rows do reach the epilogue as -0 for one sign of alpha (the bf16 store keeps the sign)
    raw = torch.empty(M, N, device="cuda", dtype=torch.bfloat16)
    neg_zero = False
    for al in (1.0, -1.0):
        g.gemm(a, b, raw, M, N, K, a_mn=a_mn, b_mn=b_mn, alpha=al, block_n=block_n)
        neg_zero |= bool((raw[:8].view(torch.int16) == -32768).any())
    assert neg_zero


# ------------------------------------------------------------------------------------------------ conv wgrad

CONV_CASES = [
    # N, Cin, H, W, Cout, R, stride
    (4, 64, 16, 16, 64, 3, 1),
    (4, 64, 16, 16, 128, 3, 2),
    (4, 128, 16, 16, 64, 1, 1),
    (4, 64, 16, 16, 128, 1, 2),
    (3, 128, 7, 7, 128, 3, 1),         # odd batch: pixel boxes overhang the image
    (5, 64, 14, 14, 64, 3, 1),
    (2, 64, 20, 12, 96, 3, 1),
    (2, 64, 16, 16, 200, 3, 1),        # Cout tail (M of the GEMM)
    (2, 96, 16, 16, 64, 3, 1),         # Cin = 96: N tail inside a 128-wide tile
]


def _nhwc(t):
    return t.to(torch.bfloat16).contiguous(memory_format=torch.channels_last)


def _wgrad_ref(x, dy, R, stride, pad):
    """float64 dW in [Cout][R][S][Cin] order, and the same on absolute values."""
    N, Cout = dy.shape[0], dy.shape[1]
    outs = []
    for xx, gg in ((x.double(), dy.double()), (x.double().abs(), dy.double().abs())):
        cols = F.unfold(xx, R, padding=pad, stride=stride)                  # [N, Cin*R*S, L]
        dw = torch.einsum("nol,nkl->ok", gg.reshape(N, Cout, -1), cols)     # [Cout, Cin*R*S]
        outs.append(dw.reshape(Cout, -1, R, R).permute(0, 2, 3, 1).contiguous())
    return outs


@pytest.mark.parametrize("N,Cin,H,W,Cout,R,stride", CONV_CASES)
def test_conv_wgrad_fp32_store_add_grid_invariant_and_bounded(N, Cin, H, W, Cout, R, stride):
    """The weight gradient written to an fp32 dw: stored for every split count and grid, then added onto a
    prior; grid-invariant bits, and within the fp64 bound."""
    lib = _conv_lib()
    gen = torch.Generator(device="cuda").manual_seed(N * H + Cout)
    pad = (R - 1) // 2
    OH, OW = H // stride, W // stride
    x = _nhwc(torch.randn(N, Cin, H, W, device="cuda", generator=gen))
    dy = _nhwc(torch.randn(N, Cout, OH, OW, device="cuda", generator=gen))
    ref64, mag64 = _wgrad_ref(x, dy, R, stride, pad)
    n_terms = N * OH * OW

    def run(splits, max_ctas, prefill=None):
        buf = torch.zeros(Cout, R, R, Cin, device="cuda", dtype=torch.float32) if prefill is None \
            else prefill.clone()
        rc = lib.b200dp_conv_wgrad(dy.data_ptr(), x.data_ptr(), buf.data_ptr(), N, H, W, Cin, Cout, R, R,
                                   stride, pad, splits, 0, max_ctas, int(prefill is not None), 0, _stream())
        assert rc == 0, lib.b200dp_conv_last_error()
        torch.cuda.synchronize()
        return buf

    for splits in (1, 2, 3, 7, 0):
        first = run(splits, 0)
        for max_ctas in (1, 5):
            again = run(splits, max_ctas)
            assert torch.equal(again, first), \
                f"splits={splits}: max_ctas={max_ctas} != default grid (max diff {float((again - first).abs().max()):.3g})"
        _assert_within_bound(first, ref64, mag64, n_terms, group="conv wgrad")
    pre = torch.randn(Cout, R, R, Cin, device="cuda", generator=gen)
    acc = run(0, 0, prefill=pre)
    _assert_within_bound(acc, pre.double() + ref64, pre.double().abs() + mag64, n_terms + 1, group="conv wgrad")


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
@pytest.mark.parametrize("N,Cin,H,W,Cout,R,stride", CONV_CASES)
def test_conv_wgrad_add_store_match_two_stage_bits(N, Cin, H, W, Cout, R, stride, dtype):
    """The weight gradient written in bf16 or fp32, added (onto a prior whose output channel 0 is -0) or
    stored, for every split count.  dy channel 0 is zero against an all-negative x, so dw[0] is a sum of
    signed zeros."""
    lib = _conv_lib()
    gen = torch.Generator(device="cuda").manual_seed(N * H + Cout + 1)
    pad = (R - 1) // 2
    OH, OW = H // stride, W // stride
    x = _nhwc(-torch.randn(N, Cin, H, W, device="cuda", generator=gen).abs())
    dy = torch.randn(N, Cout, OH, OW, device="cuda", generator=gen)
    dy[:, 0] = 0
    dy = _nhwc(dy)
    prior = torch.randn(Cout, R, R, Cin, device="cuda", generator=gen).to(dtype)
    prior[0] = -0.0

    def run(buf, splits, acc):
        rc = lib.b200dp_conv_wgrad(dy.data_ptr(), x.data_ptr(), buf.data_ptr(), N, H, W, Cin, Cout, R, R, stride,
                                   pad, splits, 0, 0, int(acc), int(buf.dtype == torch.bfloat16), _stream())
        assert rc == 0, lib.b200dp_conv_last_error()

    for splits in (1, 2, 3, 7, 0):
        for acc in (False, True):
            ref = _two_stage(lambda buf: run(buf, splits, True), prior, acc)
            out = prior.clone() if acc else torch.full_like(prior, float("nan"))
            run(out, splits, acc)
            torch.cuda.synchronize()
            _assert_same_bits(out, ref, f"splits={splits} acc={acc}")


# ------------------------------------------------------------------------------------------------ BN statistics

def _stats_ref(y2, prefill=None):
    """float64 column sums | sums of squares of the bf16 output rows y2 [M, C] (+ prefill)."""
    y = y2.double()
    ref = torch.cat([y.sum(0), (y * y).sum(0)])
    mag = torch.cat([y.abs().sum(0), (y * y).sum(0)])
    if prefill is not None:
        ref, mag = ref + prefill.double(), mag + prefill.double().abs()
    return ref, mag


# Launches of one call with these grid caps, in this order.  The output tiles do not depend on the grid,
# but the statistics do (a CTA's slot sums the tiles it ran), so the statistics are compared between
# launches with the same cap: each repeat follows launches with other grids, whose slot and arrival-counter
# state it must not inherit.
GRID_SEQUENCE = (0, 1, 7, 0, 1, 7)


def _assert_repeats(runs):
    for i, (y, st) in enumerate(runs):
        assert torch.equal(y, runs[0][0]), f"output of launch {i} depends on the grid"
        j = GRID_SEQUENCE.index(GRID_SEQUENCE[i])
        assert torch.equal(st, runs[j][1]), \
            f"max_ctas={GRID_SEQUENCE[i]}: repeated statistics differ (max diff {float((st - runs[j][1]).abs().max()):.3g})"


def test_epilogue_stats_sum_slots_in_cta_order():
    """The last CTA adds the per-CTA slots in CTA order.  With one 128-row tile per CTA (y = A @ I = A)
    and column sums 2^25 in CTA 0's tile and 1 in each later one, CTA order gives exactly 2^25 (each
    later 1 is below half an ulp of 2^25 and rounds away), any order that adds the ones first gives
    2^25 + 4."""
    g = _gemm()
    ctas, N = 5, 64
    M = 128 * ctas
    a = torch.zeros(M, N, device="cuda", dtype=torch.bfloat16)
    a[0] = 2.0 ** 25
    a[128::128] = 1.0
    eye = torch.eye(N, device="cuda", dtype=torch.bfloat16)
    y = torch.empty(M, N, device="cuda", dtype=torch.bfloat16)
    st = torch.zeros(2 * N, device="cuda", dtype=torch.float32)
    g.gemm(a, eye, y, M, N, N, stats=st, max_ctas=ctas)
    torch.cuda.synchronize()
    assert torch.equal(y, a)
    expected = torch.zeros(2 * N, device="cuda", dtype=torch.float32)
    for c in range(ctas):                      # slot c: the (exact) sums of CTA c's tile, in fp32
        t = y[128 * c:128 * (c + 1)].double()
        expected = expected + torch.cat([t.sum(0), (t * t).sum(0)]).float()
    assert float(expected[0]) == 2.0 ** 25
    assert torch.equal(st, expected), (st[:2].tolist(), expected[:2].tolist())


def test_bn_stats_sum_slots_in_block_order():
    """The same for the stand-alone reduction: block b reads rows 1024 b .. 1024 b + 1023 first (C = 8),
    and the last block adds the slots in block order, so 2^25 in block 0 absorbs the ones of blocks 1-4."""
    lib = _bn_lib()
    C, blocks = 8, 5
    x = torch.zeros(1024 * blocks, C, device="cuda", dtype=torch.bfloat16)
    x[0] = 2.0 ** 25
    x[1024::1024] = 1.0
    st = torch.zeros(2 * C, device="cuda")
    assert lib.b200dp_bn_stats(x.data_ptr(), st.data_ptr(), x.shape[0], C, _stream()) == 0
    torch.cuda.synchronize()
    assert torch.equal(st[:C], torch.full((C,), 2.0 ** 25, device="cuda")), st[:C].tolist()


GEMM_STATS_CASES = [
    # M, N, K, bias
    (1000, 256, 512, False),
    (1000, 264, 200, False),
    (1000, 200, 128, True),            # rows past M in the last tile see the bias, not zeros
    (1000, 2048, 6144, False),         # N*K*2 > 20 MB: M-fastest tile order, statistics flushed per tile
]


@pytest.mark.parametrize("M,N,K,bias", GEMM_STATS_CASES)
def test_gemm_epilogue_stats(M, N, K, bias):
    g = _gemm()
    gen = torch.Generator(device="cuda").manual_seed(M + N + K)
    a = torch.randn(M, K, device="cuda", generator=gen).to(torch.bfloat16)
    b = (torch.randn(N, K, device="cuda", generator=gen) * K ** -0.5).to(torch.bfloat16)
    bvec = (torch.randn(N, device="cuda", generator=gen) + 2.0).to(torch.bfloat16) if bias else None
    runs = []
    for max_ctas in GRID_SEQUENCE:
        y = torch.empty(M, N, device="cuda", dtype=torch.bfloat16)
        st = torch.zeros(2 * N, device="cuda", dtype=torch.float32)
        g.gemm(a, b, y, M, N, K, bias=bvec, stats=st, max_ctas=max_ctas)
        torch.cuda.synchronize()
        ref, mag = _stats_ref(y)
        _assert_within_bound(st, ref, mag, M, group="gemm epilogue stats")
        runs.append((y, st))
    _assert_repeats(runs)
    pre = torch.randn(2 * N, device="cuda", generator=gen).abs() * 10
    st = pre.clone()
    y = torch.empty(M, N, device="cuda", dtype=torch.bfloat16)
    g.gemm(a, b, y, M, N, K, bias=bvec, stats=st)
    torch.cuda.synchronize()
    ref, mag = _stats_ref(y, pre)
    _assert_within_bound(st, ref, mag, M + 1, group="gemm epilogue stats")


CONV_STATS_CASES = [
    # N, Cin, H, W, Cout, R, stride
    (3, 64, 7, 7, 128, 3, 1),
    (5, 64, 14, 14, 64, 3, 1),
    (3, 128, 14, 14, 256, 3, 2),
    (2, 64, 20, 12, 96, 3, 1),
    (3, 128, 14, 14, 256, 1, 2),
    (4, 64, 16, 16, 64, 3, 1),
]


@pytest.mark.parametrize("N,Cin,H,W,Cout,R,stride", CONV_STATS_CASES)
def test_conv_epilogue_stats(N, Cin, H, W, Cout, R, stride):
    lib = _conv_lib()
    gen = torch.Generator(device="cuda").manual_seed(N * W + Cout + R)
    pad = (R - 1) // 2
    OH, OW = H // stride, W // stride
    x = _nhwc(torch.randn(N, Cin, H, W, device="cuda", generator=gen) + 0.5)
    w = _nhwc(torch.randn(Cout, Cin, R, R, device="cuda", generator=gen) * (Cin * R * R) ** -0.5)

    def run(max_ctas, prefill=None):
        y = torch.empty(N, Cout, OH, OW, device="cuda", dtype=torch.bfloat16, memory_format=torch.channels_last)
        st = torch.zeros(2 * Cout, device="cuda", dtype=torch.float32) if prefill is None else prefill.clone()
        rc = lib.b200dp_conv_fprop(x.data_ptr(), w.data_ptr(), y.data_ptr(), N, H, W, Cin, Cout, R, R, stride,
                                   pad, 0, max_ctas, st.data_ptr(), _stream())
        assert rc == 0, lib.b200dp_conv_last_error()
        torch.cuda.synchronize()
        return y, st

    runs = []
    for max_ctas in GRID_SEQUENCE:
        y, st = run(max_ctas)
        ref, mag = _stats_ref(y.permute(0, 2, 3, 1).reshape(-1, Cout))
        _assert_within_bound(st, ref, mag, N * OH * OW, group="conv epilogue stats")
        runs.append((y, st))
    _assert_repeats(runs)
    # the output itself, against a float64 convolution of the same bf16 operands
    y = runs[0][0]
    y64 = F.conv2d(x.double(), w.double(), None, stride, pad)
    m64 = F.conv2d(x.double().abs(), w.double().abs(), None, stride, pad)
    _assert_within_bound(y, y64, m64, Cin * R * R, out_bf16=True, group="conv fprop output")
    pre = torch.randn(2 * Cout, device="cuda", generator=gen)
    y, st = run(3, prefill=pre)
    ref, mag = _stats_ref(y.permute(0, 2, 3, 1).reshape(-1, Cout), pre)
    _assert_within_bound(st, ref, mag, N * OH * OW + 1, group="conv epilogue stats")


BN_CHANNELS = [8, 16, 32, 64, 128, 256, 512, 1024, 2048]
BN_ROWS = [1, 7, 1000, 8 * 56 * 56]


@pytest.mark.parametrize("M", BN_ROWS)
@pytest.mark.parametrize("C", BN_CHANNELS)
def test_bn_standalone_reductions(C, M):
    lib = _bn_lib()
    assert lib.b200dp_bn_supported(C) == 1
    gen = torch.Generator(device="cuda").manual_seed(C + M)
    x = (3 + 0.5 * torch.randn(M, C, device="cuda", generator=gen)).to(torch.bfloat16)
    dy = (0.5 + torch.randn(M, C, device="cuda", generator=gen)).to(torch.bfloat16)
    keep = torch.rand(M, C, device="cuda", generator=gen) > 0.4
    bits = (keep.view(M, C // 8, 8).to(torch.uint8) << torch.arange(8, device="cuda", dtype=torch.uint8)).sum(
        dim=2).to(torch.uint8).contiguous()
    mean = x.float().mean(0) + 0.01 * torch.randn(C, device="cuda", generator=gen)

    def stats():
        st = torch.full((2 * C,), 123.0, device="cuda")          # the call zeroes it first
        assert lib.b200dp_bn_stats(x.data_ptr(), st.data_ptr(), M, C, _stream()) == 0
        return st

    def bwd(relu):
        s = torch.full((2 * C,), -7.0, device="cuda")
        assert lib.b200dp_bn_bwd_reduce(dy.data_ptr(), x.data_ptr(), bits.data_ptr() if relu else None,
                                        mean.data_ptr(), s.data_ptr(), M, C, int(relu), _stream()) == 0
        return s

    st = stats()
    torch.cuda.synchronize()
    ref, mag = _stats_ref(x)
    _assert_within_bound(st, ref, mag, M, group="bn stand-alone stats")
    assert torch.equal(stats(), st)
    x64, m64 = x.double(), mean.double()
    for relu in (False, True):
        s = bwd(relu)
        torch.cuda.synchronize()
        dz = dy.double() * keep.double() if relu else dy.double()
        xc = x64 - m64
        ref = torch.cat([dz.sum(0), (dz * xc).sum(0)])
        mag = torch.cat([dz.abs().sum(0), (dz.abs() * xc.abs()).sum(0)])
        _assert_within_bound(s, ref, mag, M, group="bn stand-alone bwd reduce")
        assert torch.equal(bwd(relu), s)


def test_bn_unsupported_channels_are_refused():
    """C = 96 (12 vectors of 8 channels: not a divisor of the 256-thread block) is refused by the library,
    and conv+BN falls back to the PyTorch BatchNorm instead of running the fused kernels."""
    import torch.nn as nn
    from distributed_torch_horovod_gcp_b200.ops import bn as B, counters
    lib = _bn_lib()
    C, M = 96, 64
    assert lib.b200dp_bn_supported(C) == 0
    x = torch.randn(M, C, device="cuda").to(torch.bfloat16)
    st = torch.zeros(2 * C, device="cuda")
    mean = torch.zeros(C, device="cuda")
    assert lib.b200dp_bn_stats(x.data_ptr(), st.data_ptr(), M, C, _stream()) == -1
    assert lib.b200dp_bn_bwd_reduce(x.data_ptr(), x.data_ptr(), None, mean.data_ptr(), st.data_ptr(), M, C, 0,
                                    _stream()) == -1
    torch.cuda.synchronize()
    assert float(st.abs().sum()) == 0.0
    torch.manual_seed(3)
    conv = nn.Conv2d(64, C, 3, 1, 1, bias=False).cuda().to(torch.bfloat16).to(memory_format=torch.channels_last)
    bn = nn.BatchNorm2d(C).cuda().to(torch.bfloat16)
    xi = _nhwc(torch.randn(2, 64, 12, 12, device="cuda"))
    before = counters.snapshot()
    y = B.conv_bn_act(xi, conv, bn, relu=True)
    after = counters.snapshot()
    assert after.get("bn_fwd", 0) == before.get("bn_fwd", 0), "fused BN ran for an unsupported C"
    assert getattr(bn, "_b200dp_stats", None) is None
    yc = F.conv2d(xi.float(), conv.weight.float(), None, 1, 1)
    ref = torch.relu(F.batch_norm(yc, None, None, bn.weight.float(), bn.bias.float(), True, 0.0, bn.eps))
    assert ((y.float() - ref).norm() / ref.norm()).item() < 2e-2


# ------------------------------------------------------------------------------------------------ end to end

def _bench(out_dir, steps):
    cmd = [sys.executable, os.path.join(ROOT, "bench.py"), "--model", "resnet50", "--batch", "16",
           "--image-size", "64", "--steps", str(steps), "--warmup", "1", "--no-baseline", "--no-e2e",
           "--dump-outputs", str(out_dir)]
    r = subprocess.run(cmd, cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    return np.load(os.path.join(out_dir, "loss.npy")), np.load(os.path.join(out_dir, "params_sample.npy"))


def test_resnet_step_reproducible_across_processes(tmp_path):
    l1, p1 = _bench(tmp_path / "a", 3)
    l2, p2 = _bench(tmp_path / "b", 3)
    assert np.isfinite(l1).all()
    assert np.array_equal(l1, l2), (l1, l2)
    assert np.array_equal(p1, p2), f"{int((p1 != p2).sum())} of {p1.size} parameters differ"
    _, p3 = _bench(tmp_path / "c", 4)
    assert not np.array_equal(p1, p3), "one more step left the parameters unchanged: the comparison is vacuous"


def test_resnet_step_reproducible_in_one_process(hvd_single, monkeypatch):
    """Two models built from the same seed and trained for 3 steps in the same process end bit-identical:
    no state (persistent BatchNorm statistics accumulators, reduction slots) leaks from one run into the next."""
    monkeypatch.setenv("B200DP_FUSED_SINGLE", "1")
    hvd = hvd_single
    from distributed_torch_horovod_gcp_b200.models import resnet50
    dev = torch.device("cuda", 0)
    gen = torch.Generator(device="cuda").manual_seed(11)
    batches = [(_nhwc(torch.randn(16, 3, 64, 64, device="cuda", generator=gen)),
                torch.randint(0, 100, (16,), device="cuda", generator=gen)) for _ in range(2)]

    def train():
        torch.manual_seed(1234)
        model = resnet50(num_classes=100).to(dev).to(torch.bfloat16).to(memory_format=torch.channels_last)
        model.train()
        opt = hvd.DistributedOptimizer(torch.optim.SGD(model.parameters(), lr=0.1, momentum=0.9, weight_decay=1e-4),
                                       named_parameters=model.named_parameters())
        assert opt.fused_engine is not None
        losses = []
        for i in range(3):
            x, y = batches[i % 2]
            loss = F.cross_entropy(model(x).float(), y)
            loss.backward()
            opt.step()
            opt.zero_grad()
            losses.append(loss.detach().clone())
        torch.cuda.synchronize()
        state = {k: v.detach().clone() for k, v in model.state_dict().items()}
        opt.remove_hooks()
        return torch.stack(losses), state

    l1, s1 = train()
    l2, s2 = train()
    assert torch.isfinite(l1).all()
    assert torch.equal(l1, l2), (l1.tolist(), l2.tolist())
    assert s1.keys() == s2.keys()
    differ = [k for k in s1 if not torch.equal(s1[k], s2[k])]
    assert not differ, f"{len(differ)} tensors differ, e.g. {differ[:5]}"
    assert any("running_var" in k for k in s1)
