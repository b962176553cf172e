"""Fused LM-head cross-entropy (csrc/xent_sm90.cu, ops/xent.py) on an H100.

1. Forward (per-row loss, sum, mean) and backward (dx, dW) against float64 on the exact bf16 inputs the kernels
   saw, element by element, with bounds derived from the roundings the kernels perform (``xent_fwd_bounds``,
   ``xent_grad_bounds``), in the manner of test_gpu_vit_numerics / test_gpu_causal_attention.
2. ignore_index, out-of-range targets, bitwise reproducibility, memory, the reference fall-back, CUDA graphs.
3. GPT-2 small and gpt_tiny through ``model(idx, targets)``.
"""
import math
import os
import sys

import pytest
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TESTS = os.path.dirname(os.path.abspath(__file__))
for _p in (ROOT, TESTS):
    if _p not in sys.path:
        sys.path.insert(0, _p)

from fp64_bounds import U32, U_BF16, assert_within_bound, report_ratios  # noqa: E402
from test_gpu_vit_numerics import LN2, LOG2E, U_EX2, U_LOG2  # noqa: E402

gpu = pytest.mark.gpu
TILE = 128
ROW_CHUNK = 1024          # rows per float64 reference block (keeps the [rows, V] fp64 temporaries small)


@pytest.fixture(scope="module", autouse=True)
def _report_ratios():
    yield
    report_ratios()


def _xent():
    from distributed_torch_horovod_gcp_b200.ops import kernels, xent
    assert kernels.has("linear_cross_entropy"), "xent kernels missing from libb200dp_kernels.so"
    return xent


def _F2():
    from distributed_torch_horovod_gcp_b200.ops import functional
    return functional


def xent_inputs(N, V, D, seed, ignore=()):
    """x [N, D], w [V, D] bf16 on the GPU (generated on the CPU: the same values on every machine), logits with
    standard deviation about 2; int64 targets, -100 at the rows in ``ignore``."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(N, D, generator=g).bfloat16()
    w = (torch.randn(V, D, generator=g) * (2.0 / math.sqrt(D))).bfloat16()
    t = torch.randint(0, V, (N,), generator=g)
    for i in ignore:
        if i < N:
            t[i] = -100
    return x.cuda(), w.cuda(), t.cuda()


# ================================================================================================ bounds
def _row_terms(x64, w64, t, V):
    """float64 logits z, their fp32 accumulation bound dz = 2 D u (|x| |w|^T), lse*, and the lse bound.

    The forward kernel (one row; x_j = z_j log2(e)):
    1. z~_j: fp32 accumulation of D exact bf16 products, |z~_j - z_j| <= dz_j.
    2. Each thread folds its columns into (m, s): exponent fma(z~, fl(log2 e), -m) (roundings u|x| for the
       constant and u(xmax - x + 1) for the fma), rescales ex2(m_old - m_new); then 2 quad combines and the
       fold of at most nb ranges, each one subtraction of maxima (all these together <= 6u(xmax - xmin + 1)),
       and at most 2 nb + 3 ex2.approx factors (1 + U_EX2) on any weight's path.  Relative weight error
       eta = max_j 2^E_j (1 + U_EX2)^(2 nb + 3) - 1.  No weight may flush (spread < 120 log2 units).
    3. s: fp32 adds and rescaling products, at most V + 4 nb + 8 of them on any path: eps_l.
    4. lse = (m + log2f(s)) fl(ln 2): log2f within U_LOG2 (log2 V + 1), then 4 roundings relative to |lse|."""
    nb = -(-V // TILE)
    z = x64 @ w64.T
    dz = 2 * x64.shape[1] * U32 * (x64.abs() @ w64.abs().T)
    lse = torch.logsumexp(z, dim=-1)
    xl = z * LOG2E
    xmax, xmin = xl.amax(-1, keepdim=True), xl.amin(-1, keepdim=True)
    assert float((xmax - xmin).max()) < 120.0, "a softmax weight could flush to zero: the bound does not apply"
    E = LOG2E * dz * (1 + U32) + U32 * xl.abs() + U32 * (xmax - xl + 1) + 6 * U32 * (xmax - xmin + 1)
    eta = torch.expm1(LN2 * E.amax(-1) + (2 * nb + 3) * math.log1p(U_EX2))
    assert float(eta.max()) < 0.1
    eps_l = 2 * (V + 4 * nb + 8) * U32
    c_lse = LN2 * (-torch.log2(1 - eta) - math.log2(1 - eps_l) + U_LOG2 * (math.log2(V) + 1)) * (1 + 4 * U32)
    lse_bound = c_lse + 4 * U32 * lse.abs()
    return z, dz, lse, lse_bound


def xent_fwd_bounds(x, w, t, ignore_index=-100):
    """float64 per-row losses and their bounds: loss = lse - z_t (one more rounding, and z_t's own dz)."""
    V = w.shape[0]
    w64 = w.double()
    loss, bound = [], []
    for r0 in range(0, x.shape[0], ROW_CHUNK):
        x64, tc = x[r0:r0 + ROW_CHUNK].double(), t[r0:r0 + ROW_CHUNK]
        z, dz, lse, lse_b = _row_terms(x64, w64, tc, V)
        ign = tc == ignore_index
        tt = tc.clamp(0, V - 1)[:, None]
        l = torch.where(ign, torch.zeros_like(lse), lse - z.gather(1, tt)[:, 0])
        b = torch.where(ign, torch.zeros_like(lse), (lse_b + dz.gather(1, tt)[:, 0]) * (1 + U32) + U32 * l.abs())
        loss.append(l)
        bound.append(b)
    return torch.cat(loss), torch.cat(bound)


def xent_grad_bounds(x, w, t, s, n_chunks, ignore_index=-100):
    """float64 dx, dW of sum_i s_i loss_i and their bounds.  ``s``: the exact per-row scales (0 for ignored rows).

    1. p~ = ex2(fma(z~, fl(log2 e), -lse2)), lse2 = fl(lse~ fl(log2 e)): exponent error
       E = log2(e) dz (1 + u) + u|x| + u(|x - lse2| + 1) + |lse2 - lse2*|, so |p~ - p*| <= pi p*,
       pi = (2^E - 1)(1 + U_EX2) + U_EX2 (pi = 1 where p* may flush).
    2. g~ = bf16(s~ (p~ - [j == t])): the subtraction and the product round once each, s~ = fl(grad / count) once,
       then the bf16 store (U_BF16).  G >= |g~ - g*|.
    3. dx = g~ W: fp32 over V terms, bf16 store.  dW = g~^T x: fp32 over the N rows, plus the split-K and
       chunk partial sums (< 2 N / 128 + 8 of them), one bf16 rounding."""
    V, D = w.shape
    N = x.shape[0]
    x64, w64 = x.double(), w.double()
    z, dz, lse, lse_b = _row_terms(x64, w64, t, V)
    P = torch.exp(z - lse[:, None])
    xl = z * LOG2E
    lse2 = (lse * LOG2E)[:, None]
    bl2 = (LOG2E * lse_b * (1 + U32))[:, None] + 2 * U32 * lse2.abs()
    E = LOG2E * dz * (1 + U32) + U32 * xl.abs() + U32 * ((xl - lse2).abs() + 1) + bl2
    pi = torch.expm1(LN2 * E) * (1 + U_EX2) + U_EX2
    pi = torch.where(xl - lse2 - E < -125.0, pi.clamp_min(1.0), pi)
    oh = torch.zeros_like(P)
    keep = t != ignore_index
    oh[keep] = F.one_hot(t[keep], V).double()
    s = s.double()[:, None]
    q = P - oh
    qerr = P * pi + U32 * (q.abs() + P * pi)
    G = s * q
    Gerr = (1 + U_BF16) * (s.abs() * (1 + 3 * U32) * (qerr + U32 * (q.abs() + qerr))) + U_BF16 * G.abs()
    Hm = G.abs() + Gerr
    dx = G @ w64
    dx_b = (1 + U_BF16) * (Gerr @ w64.abs() + 2 * V * U32 * (Hm @ w64.abs())) + U_BF16 * dx.abs()
    dw = G.T @ x64
    n_terms = N + 2 * (-(-N // TILE)) + n_chunks + 8
    dw_b = (1 + U_BF16) * (Gerr.T @ x64.abs() + 2 * n_terms * U32 * (Hm.T @ x64.abs())) + U_BF16 * dw.abs()
    return (dx, dx_b), (dw, dw_b)


def _sum_bounds(loss64, bound, n):
    """fp32 sum of n per-row losses in a fixed tree order: the rows' bounds plus 2 n u of the magnitudes."""
    mag = float((loss64.abs() + bound).sum())
    return float(loss64.sum()), float(bound.sum()) + 2 * n * U32 * mag


# ================================================================================================ forward
FWD_N = [1, 127, 128, 129, 8191]
FWD_V = [512, 1000, 8200, 50304]
FWD_D = [64, 768]


@gpu
@pytest.mark.parametrize("D", FWD_D)
@pytest.mark.parametrize("V", FWD_V)
@pytest.mark.parametrize("N", FWD_N)
def test_forward_vs_fp64(N, V, D):
    X = _xent()
    x, w, t = xent_inputs(N, V, D, seed=N * 7 + V + D, ignore=(0, 5, 130))
    loss64, bound = xent_fwd_bounds(x, w, t)
    rows = X.linear_cross_entropy(x, w, t, reduction="none")
    assert rows.dtype == torch.float32 and rows.shape == (N,)
    assert_within_bound(rows, loss64, group="fwd loss (none)", terms=[(1.0, bound)])
    ign = t == -100
    assert float(rows[ign].abs().sum()) == 0.0
    s_ref, s_b = _sum_bounds(loss64, bound, N)
    ssum = X.linear_cross_entropy(x, w, t, reduction="sum")
    assert ssum.dim() == 0
    assert_within_bound(ssum, torch.tensor(s_ref, dtype=torch.float64, device="cuda"), group="fwd sum",
                        terms=[(s_b, torch.ones((), dtype=torch.float64, device="cuda"))])
    cnt = int((~ign).sum())
    mean = X.linear_cross_entropy(x, w, t, reduction="mean")
    if cnt == 0:
        assert torch.isnan(mean)
    else:
        m_ref = s_ref / cnt
        m_b = s_b / cnt * (1 + U32) + U32 * (abs(m_ref) + s_b / cnt)
        assert_within_bound(mean, torch.tensor(m_ref, dtype=torch.float64, device="cuda"), group="fwd mean",
                            terms=[(m_b, torch.ones((), dtype=torch.float64, device="cuda"))])


# ================================================================================================ backward
def _fwd_bwd(x, w, t, reduction, gout=None, max_ctas=0):
    X = _xent()
    xl, wl = x.clone().requires_grad_(True), w.clone().requires_grad_(True)
    loss = X.linear_cross_entropy(xl, wl, t, reduction=reduction, max_ctas=max_ctas)
    loss.backward(gout)
    torch.cuda.synchronize()
    return loss.detach(), xl.grad, wl.grad


def _scales(t, reduction, gout, ignore_index=-100):
    keep = t != ignore_index
    if reduction == "none":
        s = gout.double().clone()
    else:
        s = torch.full(t.shape, 1.0 / int(keep.sum()), dtype=torch.float64, device=t.device)
    return torch.where(keep, s, torch.zeros_like(s))


@gpu
@pytest.mark.parametrize("chunks", ["one", "many"])
@pytest.mark.parametrize("reduction", ["mean", "none"])
@pytest.mark.parametrize("N,V,D", [(300, 1000, 64), (129, 8200, 768), (1000, 512, 768)])
def test_backward_vs_fp64(N, V, D, reduction, chunks, monkeypatch):
    X = _xent()
    if chunks == "many":
        monkeypatch.setattr(X, "_CHUNK_BYTES", 2 * TILE * V)        # 128-row chunks
        assert X.chunk_rows(V) == TILE
    n_chunks = -(-N // X.chunk_rows(V))
    x, w, t = xent_inputs(N, V, D, seed=N + V + D + 3, ignore=(1, 128, 200))
    gout = None
    if reduction == "none":
        gout = (torch.rand(N, generator=torch.Generator().manual_seed(N)) * 2 - 0.5).cuda()
    _, dx, dw = _fwd_bwd(x, w, t, reduction, gout)
    (dx64, dx_b), (dw64, dw_b) = xent_grad_bounds(x, w, t, _scales(t, reduction, gout), n_chunks)
    assert_within_bound(dx, dx64, group=f"bwd dx ({reduction}, {chunks} chunk)", terms=[(1.0, dx_b)])
    assert_within_bound(dw, dw64, group=f"bwd dW ({reduction}, {chunks} chunk)", terms=[(1.0, dw_b)])
    ign = t == -100
    assert bool((dx[ign] == 0).all())


# ================================================================================================ edges
@gpu
def test_ignored_rows_and_all_ignored():
    x, w, t = xent_inputs(256, 1000, 64, seed=5, ignore=range(0, 256, 3))
    loss, dx, _ = _fwd_bwd(x, w, t, "none", torch.ones(256, device="cuda"))
    ign = t == -100
    assert bool((loss[ign] == 0).all()) and bool((dx[ign] == 0).all())
    assert bool((dx[~ign].abs().sum(1) > 0).all())
    t_all = torch.full_like(t, -100)
    X = _xent()
    ref = F.cross_entropy(F.linear(x, w).float(), t_all)
    got = X.linear_cross_entropy(x, w, t_all)
    assert torch.isnan(ref) and torch.isnan(got)
    assert float(X.linear_cross_entropy(x, w, t_all, reduction="sum")) == 0.0


@gpu
def test_out_of_range_target_is_a_nan_row():
    N, V = 300, 1000
    x, w, t = xent_inputs(N, V, 64, seed=9, ignore=(2,))
    bad = t.clone()
    bad[7], bad[150] = V, -7
    loss_ok, dx_ok, _ = _fwd_bwd(x, w, t, "none", torch.ones(N, device="cuda"))
    loss, dx, _ = _fwd_bwd(x, w, bad, "none", torch.ones(N, device="cuda"))
    nan_rows = torch.zeros(N, dtype=torch.bool, device="cuda")
    nan_rows[[7, 150]] = True
    assert bool(torch.isnan(loss[nan_rows]).all()) and bool(torch.isnan(dx[nan_rows]).all())
    assert torch.equal(loss[~nan_rows], loss_ok[~nan_rows])
    assert torch.equal(dx[~nan_rows], dx_ok[~nan_rows])
    assert torch.isnan(_xent().linear_cross_entropy(x, w, bad))


@gpu
@pytest.mark.parametrize("chunks", ["one", "many"])
def test_two_runs_are_bit_identical(chunks, monkeypatch):
    X = _xent()
    N, V, D = 1100, 50304, 768
    if chunks == "many":
        monkeypatch.setattr(X, "_CHUNK_BYTES", 4 * TILE * 2 * V)    # 512-row chunks
    x, w, t = xent_inputs(N, V, D, seed=21, ignore=(3,))
    a = _fwd_bwd(x, w, t, "mean")
    b = _fwd_bwd(x, w, t, "mean")
    for u, v in zip(a, b):
        assert torch.equal(u.view(torch.int32) if u.dtype == torch.float32 else u.view(torch.int16),
                           v.view(torch.int32) if v.dtype == torch.float32 else v.view(torch.int16))
    # a capped grid (several items per CTA, other vocab ranges) gives the same loss up to its bound
    c = _fwd_bwd(x, w, t, "mean", max_ctas=5)
    assert abs(float(c[0]) - float(a[0])) <= 1e-5 * abs(float(a[0]))


@gpu
def test_memory_stays_within_one_chunk():
    X = _xent()
    N, D, V = 8192, 768, 50304
    x, w, t = xent_inputs(N, V, D, seed=1)
    xl, wl = x.requires_grad_(True), w.requires_grad_(True)
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    with torch.no_grad():
        X.linear_cross_entropy(xl, wl, t)
    torch.cuda.synchronize()
    nograd_peak = torch.cuda.max_memory_allocated() - base
    assert nograd_peak < 16 << 20, f"no_grad forward allocated {nograd_peak} bytes"
    torch.cuda.reset_peak_memory_stats()
    X.linear_cross_entropy(xl, wl, t).backward()
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    C = X.chunk_rows(V)
    bound = C * V * 2 + V * D * 4 + V * D * 2 + N * D * 2 + (16 << 20)
    print(f"\n[lm loss memory] N={N}: fwd+bwd peak {peak / 2**20:.1f} MiB (bound {bound / 2**20:.1f} MiB; "
          f"bf16 logits alone would be {N * V * 2 / 2**20:.1f} MiB), no_grad fwd {nograd_peak / 2**20:.2f} MiB")
    assert peak <= bound


@gpu
def test_unsupported_inputs_take_the_reference_path():
    from distributed_torch_horovod_gcp_b200.ops import counters
    F2 = _F2()
    _xent()
    for dt, V in ((torch.bfloat16, 1001), (torch.float32, 1000)):
        g = torch.Generator().manual_seed(V)
        x = torch.randn(200, 64, generator=g).to(dt).cuda()
        w = (torch.randn(V, 64, generator=g) * 0.2).to(dt).cuda()
        t = torch.randint(0, V, (200,), generator=g).cuda()
        c0 = counters.snapshot().get("xent_fwd", 0)
        got = F2.linear_cross_entropy(x, w, t)
        assert counters.snapshot().get("xent_fwd", 0) == c0, "the kernel ran on an unsupported input"
        assert torch.equal(got, F.cross_entropy(F.linear(x, w).float(), t))
    c0 = counters.snapshot().get("xent_fwd", 0)
    x, w, t = xent_inputs(200, 1000, 64, seed=4)
    F2.linear_cross_entropy(x, w, t)
    assert counters.snapshot().get("xent_fwd", 0) > c0


@gpu
def test_captures_in_a_cuda_graph():
    from distributed_torch_horovod_gcp_b200.utils.graph import GraphedStep
    X = _xent()
    x, w, t = xent_inputs(700, 8200, 768, seed=17, ignore=(0, 9))
    wl = w.clone().requires_grad_(True)

    def step(xb, tb):
        loss = X.linear_cross_entropy(xb, wl, tb)
        loss.backward()
        return loss.detach()

    gs = GraphedStep(step, [x, t], warmup=2)
    # xent forward + finish + total, one backward chunk: xent_grad and the dW GEMM (x needs no gradient)
    assert gs.kernels_per_replay == 5
    with torch.no_grad():
        eager = X.linear_cross_entropy(x, w, t)
    wr = w.clone().requires_grad_(True)
    X.linear_cross_entropy(x, wr, t).backward()
    wl.grad.zero_()
    lg = gs(x, t)
    torch.cuda.synchronize()
    assert torch.equal(lg, eager)
    assert torch.equal(wl.grad, wr.grad)


# ================================================================================================ GPT
def _rel(a, b):
    a, b = a.detach().double(), b.detach().double()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


@gpu
def test_gpt2_small_loss_and_tied_gradient():
    """model(idx, targets) against F.cross_entropy(model(idx).float(), targets) on the same weights.  The old path
    rounds each logit to bf16 (|dz| <= U_BF16 |z|), which moves lse and z_t by at most U_BF16 max_j |z_ij| each;
    both paths add fp32 rounding of at most 4 V u (max_j |z_ij| + lse_i) per row."""
    from distributed_torch_horovod_gcp_b200.models import gpt2
    from distributed_torch_horovod_gcp_b200.ops import counters
    _xent()
    torch.manual_seed(0)
    m = gpt2().cuda().to(torch.bfloat16)
    B, S = 2, 1024
    g = torch.Generator(device="cuda").manual_seed(1)
    idx = torch.randint(0, 50257, (B, S + 1), generator=g, device="cuda")
    x, y = idx[:, :-1], idx[:, 1:]
    logits = m(x)
    old = F.cross_entropy(logits.float(), y.reshape(-1))
    old.backward()
    g_old = m.wte.weight.grad.clone()
    m.zero_grad()
    c0 = counters.snapshot().get("xent_fwd", 0)
    new = m(x, y)
    new.backward()
    new, old = new.detach(), old.detach()
    torch.cuda.synchronize()
    assert counters.snapshot().get("xent_fwd", 0) > c0
    g_new = m.wte.weight.grad
    zmax = logits.detach().double().abs().amax(-1)
    lse = torch.logsumexp(logits.detach().double(), -1)
    bound = float((2 * U_BF16 * (1 + U_BF16) * zmax + 4 * 50304 * U32 * (zmax + lse.abs())).mean())
    err = abs(float(new) - float(old))
    e = _rel(g_new, g_old)
    print(f"\n[gpt2 fused loss] {float(new):.6f} vs {float(old):.6f}: |diff| {err:.3e} (bound {bound:.3e}); "
          f"wte grad rel err {e:.3e}")
    assert err <= bound
    assert e < 2e-2
    assert bool(torch.isfinite(g_new).all())


@gpu
def test_gpt_tiny_fused_adamw_step_on_the_fused_loss(hvd_single, monkeypatch):
    from distributed_torch_horovod_gcp_b200.models import gpt_tiny
    from distributed_torch_horovod_gcp_b200.utils.graph import GraphedStep
    monkeypatch.setenv("B200DP_FUSED_SINGLE", "1")
    hvd = hvd_single
    _xent()
    torch.manual_seed(0)
    m = gpt_tiny().cuda().to(torch.bfloat16)
    groups = [{"params": [p for p in m.parameters() if p.dim() >= 2], "weight_decay": 0.1},
              {"params": [p for p in m.parameters() if p.dim() < 2], "weight_decay": 0.0}]
    opt = hvd.DistributedOptimizer(torch.optim.AdamW(groups, lr=1e-3, betas=(0.9, 0.95)),
                                   named_parameters=m.named_parameters())
    assert opt.fused_engine is not None
    g = torch.Generator(device="cuda").manual_seed(2)
    x = torch.randint(0, 512, (4, 128), generator=g, device="cuda")
    y = torch.randint(0, 512, (4, 128), generator=g, device="cuda")

    def step(xb, yb):
        loss = m(xb, yb)
        loss.backward()
        opt.step()
        opt.zero_grad()
        return loss.detach()

    losses = [float(step(x, y)) for _ in range(20)]
    print(f"\n[gpt_tiny fused loss] losses {losses[0]:.4f} -> {losses[-1]:.4f}")
    assert all(math.isfinite(v) for v in losses)
    assert losses[-1] < losses[0] - 1.0
    graphed = GraphedStep(step, [x, y], warmup=2)
    with torch.no_grad():
        le = m(x, y)
    lg = graphed(x, y)
    torch.cuda.synchronize()
    torch.testing.assert_close(lg, le, rtol=1e-6, atol=0)
