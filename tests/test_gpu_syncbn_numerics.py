"""``hvd.SyncBatchNorm`` (torch/sync_batch_norm.py) at world sizes 1 to 8 on one GPU, against float64 batch norm
over the global batch.

One process plays ranks 0..N-1 one after another: ``_state.is_initialized`` / ``_state.size`` say "a world of N",
and ``mpi_ops.allreduce`` is a fake that hands rank r the fp32 sum from +0 in rank order 0..N-1 of what every rank
passed it (the one-shot kernel's arithmetic, pinned by ``test_gpu_comm_numerics.py``).  Rank r's forward needs
every rank's statistics, so a step runs in three phases, each rank starting from a fresh ``deepcopy`` of its module
in every phase:
  1. forward only: record each rank's local statistics (the fake returns them unchanged);
  2. forward with the global statistics, backward: record each rank's local backward sums;
  3. forward and backward with both global sums: the outputs that are checked.
The local sums handed to the fake must be bit-identical across the phases (the reductions are fixed-order), and a
spy on ``_SyncBNKernelFn.apply`` / ``_SyncBNFn.apply`` asserts which path ran, so a kernel case cannot silently
become a PyTorch case.

References are float64 batch norm over the concatenated global batch of the exact inputs.  The kernel path reuses
the BatchNorm bounds of ``test_gpu_resnet_numerics.py`` with the chain depth of a rank's fixed-order sum plus the
N - 1 additions of the rank-order all-reduce (its +0 is exact).  The PyTorch path (``_SyncBNFn``) computes
(x - m) is w + b in separate roundings and sums in any order; its bounds are derived below with the any-order depth
max_r M_r + N - 1.  The parameter gradients are LOCAL (each rank's rows at the global mean / invstd): each is checked
on its own, and their sum over ranks against the global float64 gradient.  Nothing is fitted to observed errors.
"""
import copy
import dataclasses
from contextlib import contextmanager
from unittest import mock

import pytest
import torch
import torch.nn.functional as F

import fp64_bounds
from fp64_bounds import U32, assert_within_bound, report_ratios
from test_gpu_comm_numerics import rank_sum
from test_gpu_resnet_numerics import (BN_EPS, _sms, bf16_store, bn_bwd_bounds, bn_fwd_bounds, bn_inputs,
                                      bn_stat_bounds, running_stats_bounds, standalone_depth)

gpu = pytest.mark.gpu


@pytest.fixture(scope="module", autouse=True)
def _report_ratios():
    yield
    report_ratios()


@dataclasses.dataclass
class Case:
    name: str
    imgs: list              # images (leading-dimension entries) per rank
    C: int
    spatial: tuple          # () for a 2-D [B, C] input
    xdtype: torch.dtype
    layout: str             # "nhwc" (channels_last), "nchw" (contiguous) or "flat" (2-D / 5-D contiguous)
    pdtype: torch.dtype
    path: str               # "kernel" or "torch"
    affine: bool = True
    track: bool = True
    train: bool = True
    momentum: float = 0.1   # None: cumulative average
    steps: int = 1

    @property
    def n(self):
        return len(self.imgs)

    def __str__(self):
        return self.name


BF16, F32, F16 = torch.bfloat16, torch.float32, torch.float16
KERNEL_CASES = [
    Case("k-n2-even-c64", [4, 4], 64, (8, 8), BF16, "nhwc", BF16, "kernel"),
    Case("k-n3-4-1-7-c8", [4, 1, 7], 8, (8, 8), BF16, "nhwc", F32, "kernel"),
    Case("k-n4-empty-c256", [2, 0, 3, 1], 256, (4, 4), BF16, "nhwc", BF16, "kernel"),
    Case("k-n8-c2048", [1] * 8, 2048, (7, 7), BF16, "nhwc", F32, "kernel"),
    Case("k-n5-cumulative-c16", [2, 5, 1, 3, 1], 16, (5, 6), BF16, "nhwc", BF16, "kernel", momentum=None, steps=2),
]
TORCH_CASES = [
    Case("t-nchw-bf16", [3, 1, 2], 16, (5, 6), BF16, "nchw", BF16, "torch"),
    Case("t-nhwc-fp32", [2, 3], 32, (4, 4), F32, "nhwc", F32, "torch"),
    Case("t-nhwc-bf16-c24", [1, 2, 2], 24, (3, 5), BF16, "nhwc", BF16, "torch"),
    Case("t-2d-empty", [3, 0, 5, 1], 5, (), F32, "flat", F32, "torch"),
    Case("t-5d", [2, 1], 8, (2, 3, 4), F32, "flat", F32, "torch"),
    Case("t-no-affine", [1, 2, 3], 8, (3, 3), F32, "nchw", F32, "torch", affine=False),
    Case("t-eval-no-tracking", [2, 1], 8, (3, 4), F32, "nchw", F32, "torch", track=False, train=False),
]


def rows(t):
    """[B, C, *spatial] (any memory layout) or [B, C] -> [B * prod(spatial), C], rows in logical order."""
    return t.movedim(1, -1).reshape(-1, t.shape[1])


def _hw(case):
    p = 1
    for s in case.spatial:
        p *= s
    return p


def _depth_f(case, sizes):
    """Chain depth of the global statistics: a rank's own sum, then N - 1 additions of the all-reduce."""
    if case.path == "kernel":
        return max(standalone_depth(m, case.C, _sms()) for m in sizes) + case.n - 1
    return max(sizes) + case.n - 1


def make_inputs(case, step, device):
    """Per-rank x and dy shards, cut from one global batch in rank order (x from ``bn_inputs``' channel mix)."""
    sizes = [b * _hw(case) for b in case.imgs]
    M = sum(sizes)
    D = _depth_f(case, sizes) + (case.path == "torch")
    g = torch.Generator().manual_seed(1000 * step + 7 * case.C + M)
    x2 = bn_inputs(M, case.C, seed=31 * step + case.C + M, D=D).float()
    dy2 = torch.randn(M, case.C, generator=g)
    if case.xdtype == F32:       # full fp32 mantissas, constant channels kept constant
        live = torch.arange(case.C) % 4 != 3
        x2[:, live] += 1e-3 * torch.randn(M, int(live.sum()), generator=g)
    else:
        dy2 = dy2 + 0.25
    x2, dy2 = x2.to(case.xdtype), dy2.to(case.xdtype)
    xs, dys, o = [], [], 0
    for b, m in zip(case.imgs, sizes):
        shard = []
        for t in (x2, dy2):
            v = t[o:o + m].reshape(b, *case.spatial, case.C).movedim(-1, 1).to(device)
            if case.layout == "nhwc":
                v = v.contiguous(memory_format=torch.channels_last)
            else:
                v = v.contiguous()
            shard.append(v)
        xs.append(shard[0])
        dys.append(shard[1])
        o += m
    return xs, dys


def make_module(case, device):
    import distributed_torch_horovod_gcp_b200.torch as hvd
    g = torch.Generator().manual_seed(case.C + case.n)
    bn = hvd.SyncBatchNorm(case.C, eps=BN_EPS, momentum=case.momentum, affine=case.affine,
                           track_running_stats=case.track)
    with torch.no_grad():
        if case.affine:
            bn.weight.copy_(torch.rand(case.C, generator=g) + 0.5)
            bn.bias.copy_(0.3 * torch.randn(case.C, generator=g))
        if case.track:
            bn.running_mean.copy_(torch.randn(case.C, generator=g))
            bn.running_var.copy_(torch.rand(case.C, generator=g) + 0.5)
    bn = bn.to(device).to(case.pdtype)
    return bn.train(case.train)


# ============================================================================================ the emulated world
def sum_reduce(r, k, local):
    """What every rank gets from the allreduce: the fp32 sum from +0 in rank order of the ranks' tensors."""
    return rank_sum([t.cpu() for t in local]).to(local[0].device)


@contextmanager
def world(N, fake, paths):
    """``_state`` reports an initialised world of N; ``mpi_ops.allreduce`` is ``fake``; every SyncBN autograd
    function that runs is appended to ``paths``."""
    from distributed_torch_horovod_gcp_b200 import _state
    from distributed_torch_horovod_gcp_b200.torch import mpi_ops
    from distributed_torch_horovod_gcp_b200.torch import sync_batch_norm as sbn
    k_apply, t_apply = sbn._SyncBNKernelFn.apply, sbn._SyncBNFn.apply

    def spy(tag, fn):
        def apply(*a):
            paths.append(tag)
            return fn(*a)
        return apply

    with mock.patch.object(_state, "is_initialized", lambda: True), \
            mock.patch.object(_state, "size", lambda: N), \
            mock.patch.object(mpi_ops, "allreduce", fake), \
            mock.patch.object(sbn._SyncBNKernelFn, "apply", spy("kernel", k_apply)), \
            mock.patch.object(sbn._SyncBNFn, "apply", spy("torch", t_apply)):
        yield


def run_step(mods, xs, dys, reduce=sum_reduce, no_sync=False):
    """One training (or eval) step of N ranks in three phases.  ``mods``: each rank's module before the step (not
    modified).  Returns, per rank, the phase-3 module, y, x.grad, and the path(s) that ran; the local sums handed to
    the allreduce are checked to be bit-identical across the phases.  ``no_sync``: run every rank's forward and
    backward under ``torch.cuda.set_sync_debug_mode("error")``."""
    from distributed_torch_horovod_gcp_b200.torch import mpi_ops
    N = len(xs)
    glob = []                    # glob[k][r]: what rank r's k-th allreduce returns (k = 0 forward, 1 backward)
    cur = [0, None]              # rank, its record of the current phase

    def fake(t, op=None, name=None, **kw):
        assert op is mpi_ops.Sum and not kw, "SyncBatchNorm all-reduces with op=Sum"
        k = len(cur[1])
        cur[1].append(t.detach().clone())
        return glob[k][cur[0]].clone() if k < len(glob) else t.clone()

    records, out = [], None
    for phase in range(3):
        record, out = [[] for _ in range(N)], []
        paths = []
        with world(N, fake, paths):
            for r in range(N):
                cur[0], cur[1] = r, record[r]
                m = copy.deepcopy(mods[r])
                x = xs[r].clone().requires_grad_(True)
                n0 = len(paths)
                if no_sync:
                    torch.cuda.set_sync_debug_mode("error")
                try:
                    y = m(x)
                    if phase > 0:
                        y.backward(dys[r])
                finally:
                    if no_sync:
                        torch.cuda.set_sync_debug_mode("default")
                out.append(dict(module=m, y=y.detach(), dx=x.grad, paths=paths[n0:]))
        records.append(record)
        if phase < 2:
            glob.append([reduce(r, phase, [record[q][phase] for q in range(N)]) for r in range(N)])
    for r in range(N):
        assert len(records[0][r]) == 1 and len(records[1][r]) == 2 and len(records[2][r]) == 2, \
            "one allreduce forward, one backward"
        assert torch.equal(records[0][r][0], records[1][r][0]) and torch.equal(records[1][r][0], records[2][r][0]), \
            f"rank {r}: local forward statistics differ between phases"
        assert torch.equal(records[1][r][1], records[2][r][1]), f"rank {r}: local backward sums differ between phases"
    return out


# ======================================================================================== bounds of the PyTorch path
def torch_xhat_err(xc, r, Em, rho):
    """xhat~ = fl(fl(x - m~) is~) against xhat* = (x - m*) r*: the difference is within Em + u (|x - m*| + Em), is~
    within rho of r*, two roundings."""
    ra = (1 + rho) * (1 + U32)
    return r * ra * (Em + U32 * (xc.abs() + Em)) + r * xc.abs() * (ra - 1)


def torch_fwd_bounds(x2, gamma, beta, D, out_bf16):
    """y of ``_SyncBNFn``: fl(fl(xhat~ w) + b) stored in x's dtype, against y* = w xhat* + b.  The product is within
    |w| (Exh + u (|xhat*| + Exh)) and the sum adds one rounding."""
    m, var, r, Em, Evar, rho = bn_stat_bounds(x2, D)
    xc = x2.double() - m
    y, E = xc * r, torch_xhat_err(xc, r, Em, rho)
    if gamma is not None:
        g = gamma.double()
        y, E = y * g, g.abs() * (E * (1 + U32) + U32 * (xc * r).abs())
    if beta is not None:
        y = y + beta.double()
        E = E + U32 * (y.abs() + E)
    return y, bf16_store(E, y) if out_bf16 else E


def torch_dx_bounds(x2, dz2, gamma, D_f, D_b, out_bf16):
    """dx of ``_SyncBNFn``: fl(fl(fl(fl(dz - k1) - fl(xhat~ k2)) is~) w), k1 = fl(G1 / n), k2 = fl(G2 / n), with
    G1 = sum dz and G2 = sum fl(dz xhat~) over the global batch (any order, depth D_b; the products add one u):
    E_G2 = sum |dz| Exh + 1.01 (D_b + 1) u sum |dz| (|xhat*| + Exh); each division one rounding (2.02 u spares a
    reciprocal); the difference three roundings; is~ within rho; the product by w one more rounding."""
    m, var, r, Em, Evar, rho = bn_stat_bounds(x2, D_f)
    x, dz = x2.double(), dz2.double()
    M = x.shape[0]
    xc = x - m
    xh, Exh = xc * r, torch_xhat_err(xc, r, Em, rho)
    S1, E1 = dz.sum(0), 1.01 * D_b * U32 * dz.abs().sum(0)
    Q = (dz * xh).sum(0)
    EQ = (dz.abs() * Exh).sum(0) + 1.01 * (D_b + 1) * U32 * (dz.abs() * (xh.abs() + Exh)).sum(0)
    k1, k2 = S1 / M, Q / M
    Ek1 = E1 / M + 2.02 * U32 * (k1.abs() + E1 / M)
    Ek2 = EQ / M + 2.02 * U32 * (k2.abs() + EQ / M)
    t = dz - k1 - xh * k2
    Et = Ek1 + xh.abs() * Ek2 + Exh * (k2.abs() + Ek2) \
        + 3.03 * U32 * (dz.abs() + k1.abs() + Ek1 + (xh.abs() + Exh) * (k2.abs() + Ek2))
    g = gamma.double() if gamma is not None else torch.ones_like(r)
    ra = (1 + rho) * (1 + U32) ** 2
    dx = g * r * t
    E = g.abs() * r * (ra * Et + (ra - 1) * t.abs())
    return dx, bf16_store(E, dx) if out_bf16 else E


def local_grad_bounds(x2, dz2, m, r, Em, rho, D, pbf16, path):
    """dgamma, dbeta of ONE rank's rows at the global m~, is~ (bounds of ``bn_stat_bounds``).  dbeta = S1 = sum dz,
    within 1.01 D u sum |dz|.  Kernel: dgamma = fl(S2 is~), S2 = sum dz fl(x - m~) within
    EP = 1.01 (D + 1) u sum |dz| (|x - m*| + Em) + Em |S1| of P* = sum dz (x - m*) (``bn_bwd_bounds``' sums).
    PyTorch: dgamma = sum fl(dz xhat~), within sum |dz| Exh + 1.01 (D + 1) u sum |dz| (|xhat*| + Exh).  Then the
    store in the parameter dtype."""
    x, dz = x2.double(), dz2.double()
    xc = x - m
    S1, E1 = dz.sum(0), 1.01 * D * U32 * dz.abs().sum(0)
    dg = (dz * xc).sum(0) * r
    if path == "kernel":
        EP = 1.01 * (D + 1) * U32 * (dz.abs() * (xc.abs() + Em)).sum(0) + Em * S1.abs()
        Edg = EP * r * (1 + rho) + dg.abs() * rho
        Edg = Edg + U32 * (dg.abs() + Edg)
    else:
        Exh = torch_xhat_err(xc, r, Em, rho)
        Edg = (dz.abs() * Exh).sum(0) + 1.01 * (D + 1) * U32 * (dz.abs() * ((xc * r).abs() + Exh)).sum(0)
    if pbf16:
        return (dg, bf16_store(Edg, dg)), (S1, bf16_store(E1, S1))
    return (dg, Edg), (S1, E1)


def torch_running_bounds(rm0, rv0, m, var, Em, Evar, M, mom, pbf16):
    """``_SyncBNFn``'s update rs.mul_(1 - mom).add_(s.to(dtype) * mom) in the parameter dtype (unit up = 2^-8 for
    bf16, u for fp32): s is rounded to the dtype first (A = E_s + up (|s*| + E_s)), then the two products and the sum
    round once each, plus fl32(mom): mom A (1 + u) + 3.03 (up + u) of the terms."""
    up = 2.0 ** -8 if pbf16 else U32
    c = M / max(M - 1, 1)
    Eunb = c * (Evar + 2.02 * U32 * (var + Evar))
    out = []
    for r0, s, Es in ((rm0, m, Em), (rv0, var * c, Eunb)):
        A = Es + up * (s.abs() + Es)
        E = mom * A * (1 + U32) + 3.03 * (up + U32) * ((1 - mom) * r0.abs() + mom * (s.abs() + A))
        out += [(1 - mom) * r0 + mom * s, E]
    return out


# ============================================================================================ the checks
def check_step(case, mods0, xs, dys, out, momentum, group=""):
    """Every rank's y, dx, local dgamma / dbeta, running statistics and num_batches_tracked after one step.  Returns
    the (got, ref, bound, group) of every comparison (asserted here)."""
    N, C = case.n, case.C
    sizes = [x.numel() // C for x in xs]
    checks = []

    def chk(got, ref, bound, name):
        checks.append((got, ref, bound, f"{group}syncbn {case.path} {name}"))
        assert_within_bound(got, ref, group=checks[-1][3], terms=[(1.0, bound)])

    for r in range(N):
        assert out[r]["paths"] == [case.path], f"rank {r} ran {out[r]['paths']}, expected the {case.path} path"
    X2 = torch.cat([rows(x) for x in xs])
    DZ2 = torch.cat([rows(d) for d in dys])
    M = X2.shape[0]
    D_f = D_b = _depth_f(case, sizes)
    m0 = mods0[0]
    gamma = m0.weight.detach() if case.affine else None
    beta = m0.bias.detach() if case.affine else None
    out_bf16 = case.xdtype == BF16
    pbf16 = case.pdtype == BF16
    if case.path == "kernel":
        D_s = D_f
        yr, yb, _, _ = bn_fwd_bounds(X2, gamma, beta, None, False, D_f)
        (dxr, dxb), _, _ = bn_bwd_bounds(X2, DZ2, gamma, D_f, D_b, pbf16)
    else:
        # the products x x and dz xhat~ round before the sum (the kernel's fma does not): one more level
        D_s = D_f + 1
        yr, yb = torch_fwd_bounds(X2, gamma, beta, D_s, out_bf16)
        dxr, dxb = torch_dx_bounds(X2, DZ2, gamma, D_s, D_b, out_bf16)
    m, var, rs, Em, Evar, rho = bn_stat_bounds(X2, D_s)
    dg_sum = db_sum = 0.0
    dg_ref = db_ref = 0.0
    o = 0
    for r in range(N):
        n, res = sizes[r], out[r]
        assert res["y"].shape == xs[r].shape and res["dx"].shape == xs[r].shape
        assert res["y"].dtype == case.xdtype and res["dx"].dtype == case.xdtype
        if n:
            chk(rows(res["y"]), yr[o:o + n], yb[o:o + n], "y")
            chk(rows(res["dx"]), dxr[o:o + n], dxb[o:o + n], "dx")
        mod = res["module"]
        if case.affine:
            D_loc = standalone_depth(n, C, _sms()) if case.path == "kernel" else max(n, 1)
            (dg, Edg), (db, Edb) = local_grad_bounds(X2[o:o + n], DZ2[o:o + n], m, rs, Em, rho, D_loc, pbf16,
                                                     case.path)
            assert mod.weight.grad.dtype == case.pdtype and mod.bias.grad.dtype == case.pdtype
            chk(mod.weight.grad, dg, Edg, "local dgamma")
            chk(mod.bias.grad, db, Edb, "local dbeta")
            dg_sum, db_sum = dg_sum + mod.weight.grad.double(), db_sum + mod.bias.grad.double()
            dg_ref, db_ref = dg_ref + dg, db_ref + db
            Eg_sum = Edg if r == 0 else Eg_sum + Edg
            Eb_sum = Edb if r == 0 else Eb_sum + Edb
        if case.track:
            m_before = mods0[r]
            rm0, rv0 = m_before.running_mean.double(), m_before.running_var.double()
            bounds = running_stats_bounds if case.path == "kernel" else torch_running_bounds
            rm, Erm, rv, Erv = bounds(rm0, rv0, m, var, Em, Evar, M, momentum, pbf16)
            chk(mod.running_mean, rm, Erm, "running_mean")
            chk(mod.running_var, rv, Erv, "running_var (unbiased, global count)")
            assert bool(torch.isfinite(mod.running_mean).all() and torch.isfinite(mod.running_var).all())
            assert int(mod.num_batches_tracked) == int(m_before.num_batches_tracked) + int(case.train)
            if r:
                assert torch.equal(mod.running_mean, out[0]["module"].running_mean) and \
                    torch.equal(mod.running_var, out[0]["module"].running_var), "ranks disagree on running stats"
        else:
            assert mod.running_mean is None and mod.num_batches_tracked is None
        o += n
    if case.affine:
        # the local gradients sum to the global one (float64 sum over ranks of the stored values)
        g_dg = (DZ2.double() * (X2.double() - m)).sum(0) * rs
        assert torch.allclose(dg_ref, g_dg, rtol=1e-9, atol=1e-9)
        chk(dg_sum, g_dg, Eg_sum, "dgamma summed over ranks")
        chk(db_sum, DZ2.double().sum(0), Eb_sum, "dbeta summed over ranks")
    return checks


def run_case(case, device, reduce=sum_reduce, no_sync=False, group=""):
    base = make_module(case, device)
    mods = [base] * case.n
    checks = []
    for step in range(case.steps):
        xs, dys = make_inputs(case, step, device)
        nbt = int(mods[0].num_batches_tracked) if case.track else 0
        momentum = case.momentum if case.momentum is not None else 1.0 / (nbt + 1)
        out = run_step(mods, xs, dys, reduce=reduce, no_sync=no_sync)
        if device != "cpu":
            torch.cuda.synchronize()
        checks += check_step(case, mods, xs, dys, out, momentum, group=group)
        mods = [o["module"] for o in out]
        for mod in mods:
            mod.zero_grad(set_to_none=True)
    return checks


# ============================================================================================ GPU tests
@gpu
@pytest.mark.parametrize("case", KERNEL_CASES + TORCH_CASES, ids=str)
def test_syncbn_emulated_world_vs_fp64(case):
    from distributed_torch_horovod_gcp_b200.ops import kernels
    assert kernels.has("bn_act")
    run_case(case, "cuda")


@gpu
def test_kernel_path_has_no_host_sync():
    """The kernel path's forward and backward never wait for the device: the global row count stays there."""
    run_case(KERNEL_CASES[1], "cuda", no_sync=True)


@gpu
@pytest.mark.parametrize("layout", ["nhwc", "nchw"])
def test_world_size_one_is_batch_norm(layout):
    """At world size 1 the module is ``F.batch_norm``, bit for bit (output, dx, dgamma, dbeta, running stats)."""
    case = Case("n1", [5], 64, (6, 6), BF16, layout, BF16, "torch")
    xs, dys = make_inputs(case, 0, "cuda")
    bn = make_module(case, "cuda")
    ref = copy.deepcopy(bn)
    paths = []
    x = xs[0].clone().requires_grad_(True)
    xr = xs[0].clone().requires_grad_(True)
    with world(1, None, paths):
        y = bn(x)
        y.backward(dys[0])
    yr = F.batch_norm(xr, ref.running_mean, ref.running_var, ref.weight, ref.bias, True, 0.1, BN_EPS)
    yr.backward(dys[0])
    assert paths == []
    for a, b in ((y, yr), (x.grad, xr.grad), (bn.weight.grad, ref.weight.grad), (bn.bias.grad, ref.bias.grad),
                 (bn.running_mean, ref.running_mean), (bn.running_var, ref.running_var)):
        assert torch.equal(a, b)


@gpu
def test_kernel_path_requires_one_parameter_dtype():
    """The kernels read weight, bias and the running statistics in the dtype of ``weight``: any other mix, and fp16,
    takes the PyTorch path.  Host check only; nothing is launched."""
    from distributed_torch_horovod_gcp_b200.torch.sync_batch_norm import _kernel_path_ok
    C = 64
    x = torch.zeros(2, C, 4, 4, device="cuda", dtype=BF16).contiguous(memory_format=torch.channels_last)

    def ok(w, b, rm, rv):
        t = lambda dt: torch.ones(C, device="cuda", dtype=dt) if dt is not None else None
        return _kernel_path_ok(x, t(w), t(b), t(rm), t(rv))

    assert ok(BF16, BF16, BF16, BF16) and ok(F32, F32, F32, F32) and ok(BF16, BF16, None, None)
    assert not ok(F16, F16, F16, F16), "fp16 parameters"
    assert not ok(BF16, F32, BF16, BF16), "bf16 weight, fp32 bias"
    assert not ok(BF16, BF16, F32, F32), "bf16 parameters, fp32 running statistics"
    assert not ok(F32, F32, BF16, F32), "fp32 parameters, one bf16 running statistic"


# ============================================================================================ CPU self-checks
CPU_CASES = [
    Case("cpu-nchw-uneven-empty", [4, 1, 7, 0], 8, (3, 3), F32, "nchw", F32, "torch"),
    Case("cpu-2d", [3, 0, 5, 1], 5, (), F32, "flat", F32, "torch"),
    Case("cpu-cumulative", [2, 3, 1], 8, (2, 2), F32, "nchw", F32, "torch", momentum=None, steps=2),
]


@pytest.mark.parametrize("case", CPU_CASES, ids=str)
def test_cpu_fallback_path_within_bounds(case):
    run_case(case, "cpu")


def _must_fail(fn, prefix, match=None):
    with pytest.raises(AssertionError, match=match):
        fn()
    for k in [k for k in fp64_bounds._WORST if k.startswith(prefix)]:
        fp64_bounds._WORST.pop(k)


def test_cpu_tightest_element_at_1_01_bound_fails():
    checks = run_case(CPU_CASES[0], "cpu", group="self-check ")
    names = set()
    for got, ref, bound, name in checks:
        if name in names:
            continue
        names.add(name)
        rel = torch.where(ref != 0, bound / ref.abs(), torch.full_like(bound, float("inf"))).reshape(-1)
        i = int(torch.argmin(rel))
        assert bound.reshape(-1)[i] > 0 and rel[i] < 1, name
        for f, fails in ((0.99, False), (1.01, True)):
            bad = got.detach().double().clone().reshape(-1)
            bad[i] = ref.reshape(-1)[i] + f * bound.reshape(-1)[i]
            bad = bad.view_as(ref)
            fn = lambda: assert_within_bound(bad, ref, group="perturbed " + name, terms=[(1.0, bound)])
            if fails:
                _must_fail(fn, "perturbed ")
            else:
                fn()
                fp64_bounds._WORST.pop("perturbed " + name, None)
    for k in [k for k in fp64_bounds._WORST if k.startswith("self-check ")]:
        fp64_bounds._WORST.pop(k)
    assert len(names) >= 8


def test_cpu_checker_rejects_per_rank_count():
    """An emulation whose forward divides by M_r N (every rank assumed to hold M_r rows) fails on an uneven split."""
    def count_bug(r, k, local):
        s = sum_reduce(r, k, local)
        if k == 0:
            s[-1] = float(local[r][-1]) * len(local)
        return s
    _must_fail(lambda: run_case(CPU_CASES[0], "cpu", reduce=count_bug, group="rejected "), "rejected ",
               match="outside the fp64 bound")


def test_cpu_checker_rejects_a_dropped_rank():
    """An allreduce that leaves out rank 2's contribution (7 of the 12 images) fails."""
    def drop_rank2(r, k, local):
        return rank_sum(local[:2] + local[3:])
    _must_fail(lambda: run_case(CPU_CASES[0], "cpu", reduce=drop_rank2, group="rejected "), "rejected ",
               match="outside the fp64 bound")
