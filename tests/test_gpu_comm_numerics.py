"""Cross-rank numerics of the communication kernels (csrc/comm_kernels.cu) at world sizes 1 to 8, on one GPU.

Every comm kernel reaches its peers only through the pointers of its argument blocks (``CommCtx.sig[]``,
``ARArgs.in[]/out[]``, ``CollArgs.src[]/dst[]``, ``BcastArgs.buf[]``) and passes exactly two ``rank_barrier``s.
So one process runs "rank r of a world of N" exactly: N ordinary device buffers stand for the peers' copies of
each symmetric buffer, every emulated rank gets its own ``CommCtx`` (own epoch counters, ``rank = r``, the N
signal pads), and before rank r's launch its pad is pre-credited with 2 for every peer and every block of the
grid, so both barriers pass without waiting.  Ranks run one after another, never concurrently (separate launches
need not be co-resident, and a barrier whose peer is not running would spin until the watchdog).

Each launch is isolated: before rank r runs, every buffer holds what it holds at the collective's opening barrier
in a real run (``Emu.isolated``).  What rank r changed is recorded, two ranks changing the same element is an
error, and the union of the changes is what a real run leaves.  Every buffer has GUARD elements past its end that
must stay bit-unchanged; outputs start as a signalling NaN the kernels never produce, so every element written is
seen as written.

Checks:
- reference (1), bit for bit: the fp32 sum from +0 in rank order 0..N-1, times the fp32 ``scale`` of the argument
  block, rounded to nearest even to the output type (torch float32 on the CPU).  A change of order, a per-rank
  pre-scale or a missed rank fails it.
- bound (2), float64: the ideal ``scale_true * sum_q g_q`` within a bound derived in ``sum_bound``.  It keeps (1)
  honest: an emulation that mirrored a wrong kernel (a bf16 accumulator, say) would break it.
- the write set of every rank, zero-on-consume, and the barrier bookkeeping: rank r adds exactly 2 to
  ``pad_t[(ch*128 + b)*8 + r]`` and to its own ``epoch[(ch*128 + b)*8 + t]`` for every peer t and block b < grid,
  and changes no other pad or epoch entry; the mailbox stays zero.
- a watchdog exit (mailbox already set, one peer not credited) writes nothing.
- zero-on-consume and the in-place copy-back happen after the closing barrier: the host plays the peers through
  host-mapped signal pads and watches rank r's input while the kernel waits there.

Not covered here: cross-GPU memory ordering (``ld.acquire.sys`` / ``red.release.sys``, ``ld.relaxed.sys`` peer
loads), NVLink itself, the NVLS kernels (multicast objects need real devices, and the switch's summation order is
not specified) and the staging loops of ``runtime/symm.py``.  The multi-GPU NCCL comparisons cover those.
"""
import ctypes
import math
import time
import zlib

import numpy as np
import pytest
import torch

import fp64_bounds
from fp64_bounds import U32, report_ratios
from test_gpu_optimizer_numerics import HYPER_FIELDS, Checker, Ev, _bits, _lw_layout, _rt, k7_ref

gpu = pytest.mark.gpu

F32, BF16, F16 = torch.float32, torch.bfloat16, torch.float16
VN = {F32: 4, BF16: 8, F16: 8}
DT_CODE = {F32: 0, BF16: 1, F16: 2}
GUARD = 64
THREADS = 512
CHANNELS, BLOCKS, RANKS = 4, 128, 8            # runtime/symm.py NUM_CHANNELS, MAX_BLOCKS, MAX_RANKS
PAD = CHANNELS * BLOCKS * RANKS
CH_USER = 1
TIMEOUT_NS = 2 * 10 ** 9
# signalling NaNs: arithmetic never produces them, so an output element that still holds one was not written
SENTINEL = {F32: 0x7FBADBAD, BF16: 0x7FAB, F16: 0x7D5A, torch.int32: -0x5A5A5A5B}
ALGO_ONESHOT, ALGO_TWOSHOT = 0, 1


@pytest.fixture(scope="module", autouse=True)
def _report_ratios():
    yield
    report_ratios()


# ============================================================================================ references (CPU)
def rank_sum(gs):
    """Reference (1) before the scale: fp32 ``acc = +0; acc += float32(g_q)`` for q = 0 .. N-1 (CPU tensors)."""
    acc = torch.zeros(gs[0].shape, dtype=torch.float32)
    for g in gs:
        acc = acc + g.float()
    return acc


def ref_exact(gs, sigma, dtype):
    """Reference (1): the rank-order fp32 sum times the fp32 scale ``sigma``, rounded to nearest even to dtype."""
    return (rank_sum(gs) * torch.tensor(sigma, dtype=torch.float32)).to(dtype)


U_OUT = {F32: 0.0, BF16: 2.0 ** -8, F16: 2.0 ** -11}       # relative rounding of the output store
TINY_OUT = {F32: 0.0, BF16: 2.0 ** -134, F16: 2.0 ** -25}  # half the subnormal spacing of the output type
OVF_OUT = {F32: 2.0 ** 128 * (1 - 2.0 ** -25), BF16: 2.0 ** 128 * (1 - 2.0 ** -9), F16: 65520.0}


def sum_bound(gs, sigma, scale_true, dtype):
    """(ideal, pre, bound) for every element with finite inputs: ideal = scale_true * sum_q g_q in float64, and
    bounds on |kernel - ideal| before (``pre``) and after (``bound``) the store to dtype.

    - The fp32 sum from +0 over N terms rounds N - 1 times (0 + g_0 is exact), and a rounded addition is within
      u of its exact result even when that is subnormal: |S^ - S| <= e1 = gamma_{N-1} sum|g|, with
      gamma_k = k u / (1 - k u), u = 2^-24.
    - The product P^ = fl(S^ sigma) is within u |S^ sigma| + 2^-150 (an fp32 subnormal result's half spacing),
      and |S^ sigma - scale_true S| <= sigma e1 + |sigma - scale_true| |S|, so
      pre = sigma e1 (1 + u) + u sigma |S| + |sigma - scale_true| |S| + 2^-150.
    - The store rounds once more: u_T (|ideal| + pre) + half the subnormal spacing of T (u_T = 2^-8 for bf16,
      2^-11 for fp16, 0 for fp32, whose store is the product itself).
    A result whose interval lies wholly past T's overflow threshold is +-inf exactly (``check_sum``)."""
    g64 = [g.double() for g in gs]
    n = len(g64)
    s = sum(g64)
    a = sum(g.abs() for g in g64)
    gam = (n - 1) * U32 / (1 - (n - 1) * U32)
    e1 = gam * a
    pre = sigma * e1 * (1 + U32) + U32 * sigma * s.abs() + abs(sigma - scale_true) * s.abs() + 2.0 ** -150
    ideal = scale_true * s
    return ideal, pre, pre + U_OUT[dtype] * (ideal.abs() + pre) + TINY_OUT[dtype]


def expected_nan(gs):
    """Where the sum is NaN: a NaN on any rank, or +inf and -inf on different ranks."""
    x = torch.stack([g.double() for g in gs])
    return torch.isnan(x).any(0) | ((x == math.inf).any(0) & (x == -math.inf).any(0))


def same_values(a, b):
    """Bit for bit, with NaN matched as NaN (its payload depends on the conversion that made it)."""
    a, b = a.cpu(), b.cpu()
    na, nb = torch.isnan(a), torch.isnan(b)
    return torch.equal(na, nb) and torch.equal(_bits(torch.where(na, torch.zeros_like(a), a)),
                                               _bits(torch.where(nb, torch.zeros_like(b), b)))


def check_sum(ck, group, out, gs, sigma, scale_true, dtype):
    """``out`` (the kernel's n elements) against reference (1) bit for bit, bound (2), and NaN exactly where the
    inputs make the sum NaN."""
    out = out.cpu()
    ck.true(f"{group} rank order", same_values(out, ref_exact(gs, sigma, dtype)), "differs from reference (1)")
    ck.true(f"{group} NaN set", torch.equal(torch.isnan(out), expected_nan(gs)), "NaN where the inputs have none")
    fin = torch.stack([torch.isfinite(g) for g in gs]).all(0)
    ideal, pre, bound = sum_bound([g[fin] for g in gs], sigma, scale_true, dtype)
    o = out[fin].double()
    over = (ideal.abs() - pre) >= OVF_OUT[dtype]                       # wholly past the threshold: inf
    maybe = ~over & ((ideal.abs() + pre) >= OVF_OUT[dtype]) & torch.isinf(o) & (torch.sign(o) == torch.sign(ideal))
    v = torch.where(over, torch.sign(ideal) * math.inf, torch.where(maybe, o, ideal))
    e = torch.where(over | maybe, torch.zeros_like(bound), bound)
    ck.bound(f"{group} fp64", o, Ev(v, e))


# ============================================================================================ inputs
def make_grads(N, n, dtype, gen, kind="mixed"):
    """Per-rank gradients (CPU tensors of dtype).  ``mixed`` cycles, element by element, through normal values,
    a wide dynamic range with cancellation across ranks, subnormals of the dtype, +-0 (all -0 on some elements),
    and independent log-uniform magnitudes; larger buffers also get a NaN on one rank, +inf and -inf on
    different ranks, and a lone +inf and -inf.  ``fp16max``: fp16 values in [6e4, 65504] on every rank."""
    if kind == "fp16max":
        return [(6e4 + 5504 * torch.rand(n, generator=gen, dtype=torch.float64)).to(dtype) for _ in range(N)]
    lo, hi = (-7.0, 4.0) if dtype == F16 else (-30.0, 20.0)
    sub = {F32: 2.0 ** -149, BF16: 2.0 ** -133, F16: 2.0 ** -24}[dtype]
    kmax = {F32: 4096, BF16: 127, F16: 1023}[dtype]
    seg = torch.arange(n) % 5
    e = lo + (hi - lo) * torch.rand(n, generator=gen, dtype=torch.float64)
    base = 10.0 ** e
    allneg0 = (torch.arange(n) % 35) == 3
    out = []
    for _ in range(N):
        g = torch.randn(n, generator=gen, dtype=torch.float64)
        sgn = torch.where(torch.rand(n, generator=gen) < 0.5, -1.0, 1.0).double()
        cancel = sgn * base + base * 2.0 ** -6 * torch.randn(n, generator=gen, dtype=torch.float64)
        subn = torch.randint(-kmax, kmax + 1, (n,), generator=gen).double() * sub
        zero = torch.where(allneg0, -0.0, sgn * 0.0)
        e2 = lo + (hi - lo) * torch.rand(n, generator=gen, dtype=torch.float64)
        wide = sgn * 10.0 ** e2
        g = torch.where(seg == 1, cancel, torch.where(seg == 2, subn, torch.where(seg == 3, zero,
                        torch.where(seg == 4, wide, g))))
        out.append(g.to(dtype))
    if n >= 40:
        out[N // 2][5] = math.nan
        out[0][10], out[N - 1][10] = math.inf, -math.inf
        out[N - 1][15] = math.inf
        out[0][20] = -math.inf
    return out


def scale_of(kind, N):
    """(the scale the argument block gets, in float64): 1, 1/N (inexact in fp32 for N = 3, 5, 6, 7) or the
    engine's gradient_predivide_factor f / N, f = 3."""
    return {"one": 1.0, "inv": 1.0 / N, "predivide": 3.0 / N}[kind]


def fp32(x):
    return float(np.float32(x))


# ============================================================================================ the emulated world
_MAILBOX = {}


def mailbox():
    """(host view, device pointer) of one host-mapped mailbox for the module."""
    if not _MAILBOX:
        lib = _rt().lib
        hp, dp = ctypes.c_uint64(0), ctypes.c_uint64(0)
        assert lib.b200dp_host_mailbox(64, ctypes.byref(hp), ctypes.byref(dp)) == 0
        _MAILBOX["host"], _MAILBOX["dev"] = (ctypes.c_int * 16).from_address(hp.value), dp.value
    return _MAILBOX["host"], _MAILBOX["dev"]


def _buf(n, dtype, data=None):
    """n elements (``data``, or the sentinel) followed by GUARD sentinel elements, on the GPU."""
    t = torch.empty(n + GUARD, dtype=dtype, device="cuda")
    t.view({4: torch.int32, 2: torch.int16, 1: torch.uint8}[t.element_size()]).fill_(SENTINEL[dtype])
    if data is not None:
        t[:n] = data.to("cuda")
    return t


class Emu:
    """N emulated ranks: N signal pads and N epoch arrays of NUM_CHANNELS * MAX_BLOCKS * MAX_RANKS counters, all
    filled with arbitrary counts so that an entry the kernel must not touch is seen if touched."""

    def __init__(self, N, seed=0):
        gen = torch.Generator().manual_seed(1000 + seed)
        self.N = N
        self.lib = _rt().lib
        self.box, dev = mailbox()
        self.pads = torch.randint(0, 1000, (N, PAD), generator=gen, dtype=torch.int32).cuda()
        self.epochs = torch.randint(0, 1000, (N, PAD), generator=gen, dtype=torch.int32).cuda()
        from distributed_torch_horovod_gcp_b200.runtime import symm as S
        self.ctx = []
        for r in range(N):
            c = S.CommCtx()
            for q in range(N):
                c.sig[q] = self.pads[q].data_ptr()
            c.epoch, c.err, c.timeout_ns, c.rank, c.world = self.epochs[r].data_ptr(), dev, TIMEOUT_NS, r, N
            self.ctx.append(c)

    def launch(self, ck, tag, r, fn, ch, grid, uncredited=None):
        """Pre-credit rank r's pad (2 from every peer, for every block of the grid; nothing from ``uncredited``),
        run ``fn(ctx)`` (a C entry point call), and check the counters it moved.  With ``uncredited`` the mailbox
        must already be set: the opening barrier then gives up after its spin limit, having added 1 everywhere."""
        pad = self.pads[r].view(CHANNELS, BLOCKS, RANKS)
        ep = self.epochs[r].view(CHANNELS, BLOCKS, RANKS)
        for t in range(self.N):
            if t != r:
                pad[ch, :grid, t] = ep[ch, :grid, t] + (0 if t == uncredited else 2)
        p0, e0 = self.pads.clone(), self.epochs.clone()
        rc = fn(self.ctx[r])
        assert rc == 0, self.lib.b200dp_comm_last_error()
        torch.cuda.synchronize()
        inc = 2 if uncredited is None else 1
        for t in range(self.N):
            if t != r:
                p0[t].view(CHANNELS, BLOCKS, RANKS)[ch, :grid, r] += inc
                e0[r].view(CHANNELS, BLOCKS, RANKS)[ch, :grid, t] += inc
        ck.true(f"{tag} signal pads", torch.equal(self.pads, p0), f"rank {r}: pad entries moved other than +{inc} "
                f"at [{ch}][b < {grid}][{r}] of every peer")
        ck.true(f"{tag} epochs", torch.equal(self.epochs, e0), f"rank {r}: epoch entries moved other than +{inc}")
        if uncredited is None:
            box = list(self.box[:4])
            assert box == [0, 0, 0, 0], f"{tag}: rank {r} set the mailbox {box}: the harness credited wrong entries"

    def isolated(self, ck, tag, bufs, fn, ch, grid, per_rank=None):
        """Run every rank from the same start state.  ``bufs``: name -> list of tensors (aliases allowed: an
        in-place buffer may appear under two names).  ``fn(r, ctx)`` launches rank r; ``per_rank(r, start)``
        checks rank r's launch before the buffers are restored.  Returns (final, owner): the start state with
        every rank's changes applied, and per element the rank that changed it (-1: none)."""
        uniq = {}
        for k, ts in bufs.items():
            for i, t in enumerate(ts):
                uniq.setdefault(t.data_ptr(), (k, i, t))
        start = {p: t.clone() for p, (_, _, t) in uniq.items()}
        final = {p: t.clone() for p, t in start.items()}
        owner = {p: torch.full(t.shape, -1, dtype=torch.int8, device="cuda") for p, t in start.items()}
        for r in range(self.N):
            for p, (_, _, t) in uniq.items():
                t.copy_(start[p])
            self.launch(ck, tag, r, lambda c: fn(r, c), ch, grid)
            if per_rank is not None:
                per_rank(r, {k: [start[t.data_ptr()] for t in ts] for k, ts in bufs.items()})
            for p, (k, i, t) in uniq.items():
                m = _bits(t) != _bits(start[p])
                ck.true(f"{tag} disjoint writes", not bool((m & (owner[p] >= 0)).any()),
                        f"{k}[{i}] written by rank {r} and an earlier rank")
                final[p][m] = t[m]
                owner[p][m] = r
        for p, (_, _, t) in uniq.items():
            t.copy_(final[p])
        return ({k: [final[t.data_ptr()] for t in ts] for k, ts in bufs.items()},
                {k: [owner[t.data_ptr()] for t in ts] for k, ts in bufs.items()})


def _stream():
    return torch.cuda.current_stream().cuda_stream


def ar_args(inp, out, n, scale, ch, zero_input=0, scratch=None):
    from distributed_torch_horovod_gcp_b200.runtime import symm as S
    a = S.ARArgs()
    for q in range(len(inp)):
        a.inp[q], a.out[q] = inp[q].data_ptr(), out[q].data_ptr()
    a.n, a.scale, a.channel, a.zero_input = n, scale, ch, zero_input
    if scratch is not None:
        a.scratch, a.copy_back = scratch.data_ptr(), 1
    return a


def slice_owner(n, vn, N):
    """Per element of a two-shot bucket, the rank whose slice holds it: per = ceil(nvec / N) vectors each."""
    nvec = n // vn
    per = -(-nvec // N)
    return (torch.arange(n, device="cuda") // vn) // per


def owned_by(owner, want):
    """``owner`` (int8) equals ``want`` over [0, len(want)) and is -1 (untouched) on the guard."""
    m = len(want)
    return torch.equal(owner[:m].long(), want.long()) and bool((owner[m:] == -1).all())


# ============================================================================================ all-reduce K1 / K2
AR_SIZES = ("one", "few", "odd", "k1edge-", "k1edge+", "k2edge-", "k2edge+")


def ar_nvec(size, N, grid, threads):
    return {"one": 1, "few": max(N - 1, 1), "odd": 37 * N + 3,
            "k1edge-": grid * threads - 1, "k1edge+": grid * threads + 1,
            "k2edge-": 2 * grid * threads * N - 1, "k2edge+": 2 * grid * threads * N + 1}[size]


def _ar_cases():
    cases, i = [], 0
    dts, grids, scales = (F32, BF16, F16), (1, 7, 128), ("one", "inv", "predivide")
    for N in range(2, 9):
        for d in dts:
            size = AR_SIZES[i % len(AR_SIZES)]
            grid = grids[(i // 2) % 3] if not size.startswith("k2") or N < 6 else 7
            cases.append((f"w{N}-{str(d)[6:]}-{size}-g{grid}-{scales[i % 3]}", N, d, grid, THREADS, CH_USER,
                          ar_nvec(size, N, grid, THREADS), scales[i % 3], "mixed"))
            i += 1
    cases += [
        ("w1-f32-odd-g7", 1, F32, 7, THREADS, CH_USER, 41, "one", "mixed"),
        ("w8-f16-6e4-g7-inv", 8, F16, 7, THREADS, CH_USER, 7 * THREADS + 5, "inv", "fp16max"),
        ("w8-bf16-32thr", 8, BF16, 7, 32, CH_USER, 2 * 7 * 32 * 8 + 3, "inv", "mixed"),
        ("w8-f32-ch3-g128", 8, F32, 128, THREADS, 3, 128 * THREADS + 9, "predivide", "mixed"),
        ("w6-bf16-big-g128", 6, BF16, 128, THREADS, CH_USER, 3 * (1 << 20) // 8 + 11, "inv", "mixed"),
        ("w7-f16-few-g1", 7, F16, 1, THREADS, CH_USER, 3, "inv", "mixed"),
        ("w5-f32-one-g128", 5, F32, 128, THREADS, CH_USER, 1, "predivide", "mixed"),
    ]
    return cases


AR_CASES = _ar_cases()


@gpu
@pytest.mark.parametrize("case", AR_CASES, ids=[c[0] for c in AR_CASES])
def test_allreduce(case):
    """K1 one-shot (out of place with zero_input, and in place through scratch + copy-back) and K2 two-shot (out
    of place with zero_input, in place isolated and in place sequential), OPT_NONE, on the same inputs."""
    name, N, dtype, grid, threads, ch, nvec, skind, values = case
    vn, dc = VN[dtype], DT_CODE[dtype]
    n = nvec * vn
    gen = torch.Generator().manual_seed(zlib.crc32(name.encode()))
    gs = make_grads(N, n, dtype, gen, values)
    scale_true = scale_of(skind, N)
    sigma = fp32(scale_true)
    emu = Emu(N, seed=nvec)
    lib = emu.lib
    ck = Checker()
    zeros = torch.zeros(n, dtype=dtype, device="cuda")
    ref = ref_exact(gs, sigma, dtype).cuda()

    def launcher(algo, inp, out, zero_input, scratch=None):
        def fn(r, ctx):
            a = ar_args(inp, out, n, scale_true, ch, zero_input, None if scratch is None else scratch[r])
            return lib.b200dp_comm_allreduce(ctypes.byref(ctx), ctypes.byref(a), algo, dc, grid, threads, _stream())
        return fn

    def fresh():
        return [_buf(n, dtype, g) for g in gs]

    def outs():
        return [_buf(n, dtype) for _ in range(N)]

    own = torch.arange(N, device="cuda")
    # K1 out of place, zero_input: rank q writes out[q] (the reference) and zeroes in[q], nothing else
    inp, out = fresh(), outs()
    fin, owner = emu.isolated(ck, "K1", {"in": inp, "out": out}, launcher(ALGO_ONESHOT, inp, out, 1), ch, grid)
    check_sum(ck, f"K1 {str(dtype)[6:]}", fin["out"][0][:n], gs, sigma, scale_true, dtype)
    for q in range(N):
        ck.same_bits("K1 ranks agree", fin["out"][q][:n], fin["out"][0][:n])
        ck.true("K1 out write set", owned_by(owner["out"][q], own[q].expand(n)), f"out[{q}]")
        ck.same_bits("K1 zero_input", fin["in"][q][:n], zeros)
        ck.true("K1 input write set", bool((owner["in"][q][n:] == -1).all()) and
                bool(((owner["in"][q][:n] == q) | (owner["in"][q][:n] == -1)).all()), f"in[{q}]")
    k1 = fin["out"][0][:n].clone()
    ck.true("K1 output", same_values(k1, ref), "K1 differs from reference (1)")
    # K1 in place: scratch + copy_back as SymmRuntime._ar_symm sets it up; in[q] ends up holding the result
    buf = fresh()
    scratch = outs()
    fin, owner = emu.isolated(ck, "K1 in place", {"buf": buf, "scratch": scratch},
                              launcher(ALGO_ONESHOT, buf, buf, 0, scratch), ch, grid)
    for q in range(N):
        ck.true("K1 in place result", same_values(fin["buf"][q][:n], k1), f"buf[{q}]")
        ck.true("K1 in place write set", bool((owner["buf"][q][n:] == -1).all()) and
                bool(((owner["buf"][q][:n] == q) | (owner["buf"][q][:n] == -1)).all()) and
                owned_by(owner["scratch"][q], own[q].expand(n)), f"rank {q}")
    # K2 out of place, zero_input: rank r pushes slice r into every out[q]; in[r] is zeroed over [0, nvec)
    so = slice_owner(n, vn, N)
    inp, out = fresh(), outs()
    fin, owner = emu.isolated(ck, "K2", {"in": inp, "out": out}, launcher(ALGO_TWOSHOT, inp, out, 1), ch, grid)
    for q in range(N):
        ck.true("K2 equals K1", same_values(fin["out"][q][:n], k1), f"out[{q}]")
        ck.true("K2 out write set", owned_by(owner["out"][q], so), f"out[{q}]")
        ck.same_bits("K2 zero_input", fin["in"][q][:n], zeros)
        ck.true("K2 input write set", bool((owner["in"][q][n:] == -1).all()) and
                bool(((owner["in"][q][:n] == q) | (owner["in"][q][:n] == -1)).all()), f"in[{q}]")
    # K2 in place with zero_input: nothing is zeroed (in == out); sequential launches on shared buffers
    # (without zero_input) are equivalent here because the slices are disjoint
    buf = fresh()
    fin, owner = emu.isolated(ck, "K2 in place", {"buf": buf}, launcher(ALGO_TWOSHOT, buf, buf, 1), ch, grid)
    for q in range(N):
        ck.true("K2 in place equals K1", same_values(fin["buf"][q][:n], k1), f"buf[{q}]")
        ck.true("K2 in place write set", bool((owner["buf"][q][n:] == -1).all()) and
                bool(((owner["buf"][q][:n] == so) | (owner["buf"][q][:n] == -1)).all()), f"buf[{q}]")
    seq = fresh()
    fn = launcher(ALGO_TWOSHOT, seq, seq, 0)
    for r in range(N):
        emu.launch(ck, "K2 sequential", r, lambda c: fn(r, c), ch, grid)
    for q in range(N):
        ck.same_bits("K2 sequential equals isolated", seq[q], fin["buf"][q])
    if values == "fp16max":
        ck.true("fp16 sum past 65504 stays finite", bool(torch.isfinite(k1).all()), "inf in the output")
    ck.close()


# ============================================================================================ reduce-scatter
RS_CASES = [  # id, N, dtype, grid, chunk in vectors
    ("w2-f32-edge-", 2, F32, 7, 2 * 7 * THREADS - 1), ("w3-bf16-edge+", 3, BF16, 1, 2 * THREADS + 1),
    ("w4-f16-one", 4, F16, 128, 1), ("w5-f32-odd", 5, F32, 128, 2 * 128 * THREADS + 1),
    ("w6-bf16-odd", 6, BF16, 7, 333), ("w7-f16-edge-", 7, F16, 7, 2 * 7 * THREADS - 1),
    ("w8-bf16-edge+", 8, BF16, 7, 2 * 7 * THREADS + 1),
]


@gpu
@pytest.mark.parametrize("case", RS_CASES, ids=[c[0] for c in RS_CASES])
def test_reduce_scatter(case):
    """Rank r's dst is reference (1) over chunk r of the staged inputs ``src[q] + r * chunk`` (chunk in elements),
    and nothing past the chunk or in any src is written."""
    name, N, dtype, grid, cvec = case
    from distributed_torch_horovod_gcp_b200.runtime import symm as S
    vn = VN[dtype]
    chunk = cvec * vn
    gen = torch.Generator().manual_seed(zlib.crc32(name.encode()))
    gs = make_grads(N, N * chunk, dtype, gen)
    emu, ck = Emu(N, seed=cvec), Checker()
    src, dst = [_buf(N * chunk, dtype, g) for g in gs], [_buf(chunk, dtype) for _ in range(N)]
    sigma = fp32(1.0 / N)

    def fn(r, ctx):
        a = S.CollArgs()
        for q in range(N):
            a.src[q], a.dst[q] = src[q].data_ptr(), dst[q].data_ptr()
        a.chunk, a.scale, a.channel = chunk, 1.0 / N, CH_USER
        return emu.lib.b200dp_comm_collective(ctypes.byref(ctx), ctypes.byref(a), S.COLL_REDUCE_SCATTER,
                                              DT_CODE[dtype], grid, THREADS, _stream())
    fin, owner = emu.isolated(ck, "reduce-scatter", {"src": src, "dst": dst}, fn, CH_USER, grid)
    for r in range(N):
        check_sum(ck, f"reduce-scatter {str(dtype)[6:]}", fin["dst"][r][:chunk],
                  [g[r * chunk:(r + 1) * chunk] for g in gs], sigma, 1.0 / N, dtype)
        ck.true("reduce-scatter write set", owned_by(owner["dst"][r], torch.full((chunk,), r, device="cuda")) and
                bool((owner["src"][r] == -1).all()), f"rank {r}")
    ck.close()


# ============================================================================================ all-gather / all-to-all
def pattern(r, j, nvec):
    """16-byte vectors as int32 words that name (source rank r, sub-chunk j, vector, word): no two alike."""
    w = torch.arange(nvec * 4, dtype=torch.int32, device="cuda") % (1 << 22)
    return ((r + 1) << 27) | (j << 22) | w


COPY_CASES = [("w2-g1", 2, 1, 1), ("w3-g7", 3, 7, 7 * THREADS + 1), ("w5-g128", 5, 128, 333),
              ("w6-g7", 6, 7, 1), ("w7-g128", 7, 128, 128 * THREADS - 1), ("w8-g7", 8, 7, 7 * THREADS - 1),
              ("w4-g1", 4, 1, THREADS + 1)]


@gpu
@pytest.mark.parametrize("mode", ["allgather", "alltoall"])
@pytest.mark.parametrize("case", COPY_CASES, ids=[c[0] for c in COPY_CASES])
def test_copy_collectives(case, mode):
    """All-gather: slot r of every peer's dst <- rank r's source.  All-to-all: slot r of peer j's dst <- rank r's
    sub-chunk j.  ``chunk`` counts 16-byte vectors; everything else stays as it was, byte for byte."""
    name, N, grid, nvec = case
    from distributed_torch_horovod_gcp_b200.runtime import symm as S
    emu, ck = Emu(N, seed=nvec), Checker()
    i32 = torch.int32
    subs = 1 if mode == "allgather" else N
    src = [_buf(subs * nvec * 4, i32, torch.cat([pattern(r, j, nvec) for j in range(subs)])) for r in range(N)]
    dst = [_buf(N * nvec * 4, i32) for _ in range(N)]

    def fn(r, ctx):
        a = S.CollArgs()
        for q in range(N):
            a.src[q], a.dst[q] = src[q].data_ptr(), dst[q].data_ptr()
        a.chunk, a.channel = nvec, CH_USER
        m = S.COLL_ALLGATHER if mode == "allgather" else S.COLL_ALLTOALL
        return emu.lib.b200dp_comm_collective(ctypes.byref(ctx), ctypes.byref(a), m, 0, grid, THREADS, _stream())
    fin, owner = emu.isolated(ck, mode, {"src": src, "dst": dst}, fn, CH_USER, grid)
    slots = torch.arange(N, device="cuda").repeat_interleave(nvec * 4)
    for j in range(N):
        want = torch.cat([pattern(r, 0 if mode == "allgather" else j, nvec) for r in range(N)])
        ck.same_bits(f"{mode} slots", fin["dst"][j][:N * nvec * 4], want)
        ck.true(f"{mode} write set", owned_by(owner["dst"][j], slots) and bool((owner["src"][j] == -1).all()),
                f"rank {j}")
    ck.close()


# ============================================================================================ broadcast
@gpu
@pytest.mark.parametrize("N,grid,nvec", [(2, 1, 1), (3, 7, 7 * THREADS + 3), (5, 128, 129), (8, 7, 2 * THREADS - 1)])
def test_broadcast(N, grid, nvec):
    """For every root: every other rank's buffer becomes the root's, the root's own buffer is not written, and a
    non-root launch writes nothing."""
    from distributed_torch_horovod_gcp_b200.runtime import symm as S
    emu, ck = Emu(N, seed=nvec), Checker()
    for root in range(N):
        buf = [_buf(nvec * 4, torch.int32, pattern(q, 0, nvec)) for q in range(N)]

        def fn(r, ctx):
            a = S.BcastArgs()
            for q in range(N):
                a.buf[q] = buf[q].data_ptr()
            a.nbytes, a.root, a.channel = nvec * 16, root, CH_USER
            return emu.lib.b200dp_comm_broadcast(ctypes.byref(ctx), ctypes.byref(a), grid, THREADS, _stream())
        fin, owner = emu.isolated(ck, "broadcast", {"buf": buf}, fn, CH_USER, grid)
        for q in range(N):
            ck.same_bits("broadcast values", fin["buf"][q][:nvec * 4], pattern(root, 0, nvec))
            want = torch.full((nvec * 4,), -1 if q == root else root, device="cuda")
            ck.true("broadcast write set", owned_by(owner["buf"][q], want), f"root {root}, buffer {q}")
    ck.close()


# ============================================================================================ K1c / K10 reductions
@gpu
@pytest.mark.parametrize("N,dtype,grid,nvec", [(2, F32, 7, 7 * THREADS + 1), (3, BF16, 128, 333), (5, F16, 1, 37),
                                                (7, BF16, 7, 2 * 7 * THREADS - 1), (8, F32, 128, 128 * THREADS + 3)])
def test_clip_reduction(N, dtype, grid, nvec):
    """K1c at world N: the fp32 arena r is reference (1) before its final rounding, bit for bit, on every rank;
    the per-CTA norm slots are bitwise identical on every rank (the global norm needs the same bits everywhere);
    slots past the grid, the output bucket and the peers' gradients are untouched; in[r] is zeroed."""
    from distributed_torch_horovod_gcp_b200.runtime import symm as S
    vn, n = VN[dtype], nvec * VN[dtype]
    gen = torch.Generator().manual_seed(nvec)
    gs = make_grads(N, n, dtype, gen)
    emu, ck = Emu(N, seed=nvec), Checker()
    inp, out = [_buf(n, dtype, g) for g in gs], [_buf(n, dtype) for _ in range(N)]
    r32 = [_buf(n, F32) for _ in range(N)]
    slots = [_buf(S.MAX_BLOCKS, F32) for _ in range(N)]
    scale = 1.0 / N

    def fn(r, ctx):
        a = ar_args(inp, out, n, scale, CH_USER, 1)
        k = S.ClipArgs()
        k.r, k.slots = r32[r].data_ptr(), slots[r].data_ptr()
        return emu.lib.b200dp_comm_clip_bucket(ctypes.byref(ctx), ctypes.byref(a), ctypes.byref(k), S.CLIP_REDUCE,
                                               DT_CODE[dtype], grid, THREADS, _stream())
    fin, owner = emu.isolated(ck, "K1c", {"in": inp, "out": out, "r": r32, "slots": slots}, fn, CH_USER, grid)
    want = rank_sum(gs) * torch.tensor(fp32(scale), dtype=torch.float32)
    check_sum(ck, "K1c r", fin["r"][0][:n], gs, fp32(scale), scale, F32)
    for q in range(N):
        ck.true("K1c r", same_values(fin["r"][q][:n], want), f"rank {q}")
        ck.same_bits("K1c slots agree", fin["slots"][q][:grid], fin["slots"][0][:grid])
        ck.true("K1c write set", owned_by(owner["r"][q], torch.full((n,), q, device="cuda")) and
                owned_by(owner["slots"][q], torch.full((grid,), q, device="cuda")) and
                bool((owner["out"][q] == -1).all()), f"rank {q}")
        ck.same_bits("K1c zero_input", fin["in"][q][:n], torch.zeros(n, dtype=dtype, device="cuda"))
    ck.close()


@gpu
@pytest.mark.parametrize("N,dtype,grid", [(2, BF16, 7), (4, F32, 1), (6, F16, 128), (8, BF16, 7)])
def test_layerwise_reduction(N, dtype, grid):
    """K10 (LARS, weight_decay = 0, so the direction is the reduced gradient exactly) at world N: the fp32 arena
    r is reference (1) before its final rounding on every rank, the per-chunk partial sums are bitwise identical
    on every rank, and each rank zeroes its own chunk vectors only."""
    from distributed_torch_horovod_gcp_b200.runtime import symm as S
    n, _, rows = _lw_layout(dtype, [3 * 16384 + 5, 100, 7, 16384])
    nch = len(rows)
    gen = torch.Generator().manual_seed(N)
    gs = [torch.randn(n, generator=gen).to(dtype) for _ in range(N)]
    p = torch.randn(n, generator=gen)
    emu, ck = Emu(N, seed=n), Checker()
    chunks = torch.tensor(rows, dtype=torch.int32, device="cuda")
    master = dtype != F32
    inp = [_buf(n, dtype, g) for g in gs]
    out = [_buf(n, dtype, p.to(dtype)) for _ in range(N)]
    M = [_buf(n, F32, p) for _ in range(N)] if master else []
    r32, part = [_buf(n, F32) for _ in range(N)], [_buf(2 * nch, F32) for _ in range(N)]

    def fn(r, ctx):
        a = ar_args(inp, out, n, 1.0 / N, CH_USER, 1)
        a.master = M[r].data_ptr() if master else 0
        a.h.kind, a.h.lr, a.h.momentum = S.OPT_LARS, 0.5, 0.9
        k = S.LwArgs()
        k.r, k.part, k.chunks, k.nchunks = r32[r].data_ptr(), part[r].data_ptr(), chunks.data_ptr(), nch
        k.adaptive, k.trust_coef = 1, 0.02
        return emu.lib.b200dp_comm_lw_bucket(ctypes.byref(ctx), ctypes.byref(a), ctypes.byref(k), S.LW_REDUCE,
                                             DT_CODE[dtype], grid, THREADS, _stream())
    bufs = {"in": inp, "out": out, "r": r32, "part": part, **({"M": M} if master else {})}
    fin, owner = emu.isolated(ck, "K10", bufs, fn, CH_USER, grid)
    want = rank_sum(gs) * torch.tensor(fp32(1.0 / N), dtype=torch.float32)
    for q in range(N):
        ck.true("K10 r", same_values(fin["r"][q][:n], want), f"rank {q}")
        ck.same_bits("K10 partials agree", fin["part"][q][:2 * nch], fin["part"][0][:2 * nch])
        ck.true("K10 write set", owned_by(owner["r"][q], torch.full((n,), q, device="cuda")) and
                owned_by(owner["part"][q], torch.full((2 * nch,), q, device="cuda")) and
                bool((owner["out"][q] == -1).all()) and (not master or bool((owner["M"][q] == -1).all())),
                f"rank {q}")
        ck.same_bits("K10 zero_input", fin["in"][q][:n], torch.zeros(n, dtype=dtype, device="cuda"))
    ck.close()


# ============================================================================================ fused optimizer
OPT_CASES = [  # id, N, dtype, kind, grid, nvec
    ("w2-f32-sgd", 2, F32, "sgd", 7, 7 * THREADS + 37), ("w3-bf16-adam", 3, BF16, "adam", 7, 2 * 7 * THREADS * 3 + 1),
    ("w4-f32-adam", 4, F32, "adam", 128, 333), ("w5-bf16-sgd-few", 5, BF16, "sgd", 1, 3),
    ("w6-bf16-sgd", 6, BF16, "sgd", 128, 128 * THREADS + 7), ("w7-f32-adam", 7, F32, "adam", 1, 2 * THREADS * 7 - 1),
    ("w8-bf16-adam", 8, BF16, "adam", 7, 37 * 8 + 5),
]
OPT_HYPER = {"sgd": dict(kind=1, lr=0.5, momentum=0.9, dampening=0.3, weight_decay=1e-2),
             "adam": dict(kind=2, lr=0.25, beta1=0.9, beta2=0.999, eps=1e-8, weight_decay=1e-2)}


@gpu
@pytest.mark.parametrize("case", OPT_CASES, ids=[c[0] for c in OPT_CASES])
def test_fused_optimizer(case):
    """K1 and K2 with the K7 epilogue at world N, side by side, for 3 steps from zero optimizer state.  Every
    rank's update against ``k7_ref`` fed with reference (1)'s fp32 sum and the fp32 scale, from the state that
    rank held; all ranks hold the same parameters; two-shot parameters equal one-shot ones bit for bit; under
    two-shot each rank's master / S0 / S1 change on its own slice only and S0 / S1 stay zero elsewhere, and the
    fp32 sum of the shards (what ``FusedEngine.export_state`` computes) equals the one-shot state; step counters
    +1 and tickets back to 0 on every rank, empty-slice ranks included."""
    name, N, dtype, kind, grid, nvec = case
    vn, n = VN[dtype], nvec * VN[dtype]
    gen = torch.Generator().manual_seed(nvec)
    p = torch.randn(n, generator=gen)
    master = dtype != F32
    hyper = OPT_HYPER[kind]
    scale = 1.0 / N
    so = slice_owner(n, vn, N)
    emu = Emu(N, seed=nvec)

    def state():
        st = {"in": [_buf(n, dtype, torch.zeros(n)) for _ in range(N)],
              "out": [_buf(n, dtype, p.to(dtype)) for _ in range(N)],
              "S0": [_buf(n, F32, torch.zeros(n)) for _ in range(N)],
              "S1": [_buf(n, F32, torch.zeros(n)) for _ in range(N)],
              "ints": [torch.tensor([0, 0] + [-7] * 6, dtype=torch.int32, device="cuda") for _ in range(N)]}
        if master:
            st["M"] = [_buf(n, F32, p) for _ in range(N)]
        return st

    runs = {ALGO_ONESHOT: state(), ALGO_TWOSHOT: state()}
    for step in range(3):
        gs = make_grads(N, n, dtype, gen, "mixed")
        gs = [torch.where(torch.isfinite(g), g, torch.zeros_like(g)) for g in gs]     # the optimizer sees finite
        S_hat = rank_sum(gs).double().cuda()
        fins, owners = {}, {}
        for algo, st in runs.items():
            for q in range(N):
                st["in"][q][:n] = gs[q].cuda()
            ck = Checker()
            tag = f"{'K1' if algo == ALGO_ONESHOT else 'K2'} {kind} step {step}"

            def fn(r, ctx, st=st, algo=algo):
                from distributed_torch_horovod_gcp_b200.runtime import symm as S
                a = ar_args(st["in"], st["out"], n, scale, CH_USER, 1)
                a.master = st["M"][r].data_ptr() if master else 0
                a.s0, a.s1 = st["S0"][r].data_ptr(), st["S1"][r].data_ptr() if kind == "adam" else 0
                a.step_ctr, a.ticket = st["ints"][r].data_ptr(), st["ints"][r].data_ptr() + 4
                for k, v in hyper.items():
                    setattr(a.h, k, v)
                return emu.lib.b200dp_comm_allreduce(ctypes.byref(ctx), ctypes.byref(a), algo, DT_CODE[dtype], grid,
                                                     THREADS, _stream())
            start = {k: [t.clone() for t in v] for k, v in st.items()}
            fin, owner = emu.isolated(ck, tag, st, fn, CH_USER, grid)
            from distributed_torch_horovod_gcp_b200.runtime import symm as S
            hp = S.OptHyper()
            for k, v in hyper.items():
                setattr(hp, k, v)
            h = {k: getattr(hp, k) for k in HYPER_FIELDS}
            for r in range(N):
                sl = (so == r) if algo == ALGO_TWOSHOT else torch.ones(n, dtype=torch.bool, device="cuda")
                pm = (start["M"] if master else start["out"])[r][:n].double()
                ref = k7_ref(S_hat[sl], pm[sl], start["S0"][r][:n][sl].double(), start["S1"][r][:n][sl].double(),
                             h, step, h["lr"], fp32(scale))
                got = (fin["M"] if master else fin["out"])[r][:n]
                ck.bound(f"{tag} master", got[sl], ref["p"])
                ck.bound(f"{tag} S0", fin["S0"][r][:n][sl], ref["s0"])
                if kind == "adam":
                    ck.bound(f"{tag} S1", fin["S1"][r][:n][sl], ref["s1"])
                for k in ("S0", "S1") + (("M",) if master else ()):
                    ck.true(f"{tag} {k} write set", bool((owner[k][r][:n][~sl] == -1).all()) and
                            bool((owner[k][r][n:] == -1).all()), f"rank {r} wrote {k} outside its slice")
                ck.same_bits(f"{tag} ranks agree", fin["out"][r][:n], fin["out"][0][:n])
                if master:
                    ck.same_bits(f"{tag} store", fin["out"][r][:n][sl], fin["M"][r][:n][sl].to(dtype))
                ck.same_bits(f"{tag} zero_input", fin["in"][r][:n], torch.zeros(n, dtype=dtype, device="cuda"))
                ints = fin["ints"][r].tolist()
                ck.true(f"{tag} step counter", ints == [step + 1, 0] + [-7] * 6, f"rank {r}: {ints}")
            ck.close()
            fins[algo], owners[algo] = fin, owner
        one, two = fins[ALGO_ONESHOT], fins[ALGO_TWOSHOT]
        ck = Checker()
        ck.same_bits(f"two-shot equals one-shot step {step}", two["out"][0], one["out"][0])
        for k in ("S0", "S1") if kind == "adam" else ("S0",):
            shard_sum = rank_sum([t[:n].cpu() for t in two[k]])           # fp32, rank order, as a Sum-allreduce
            ck.same_bits(f"two-shot {k} shards sum to one-shot step {step}", shard_sum, one[k][0][:n].cpu())
            for r in range(N):
                ck.true(f"two-shot {k} zero outside slice", bool((two[k][r][:n][so != r] == 0).all()), f"rank {r}")
        if master:
            for r in range(N):
                ck.same_bits(f"two-shot master slice step {step}", two["M"][r][:n][so == r], one["M"][0][:n][so == r])
        ck.close()


# ============================================================================================ watchdog exit
WD_KERNELS = ["oneshot", "twoshot", "clip", "layerwise", "reduce-scatter", "allgather", "alltoall", "broadcast"]


@gpu
@pytest.mark.parametrize("kernel", WD_KERNELS)
def test_watchdog_exit_writes_nothing(kernel):
    """With the mailbox already set and one peer not credited, the opening barrier gives up after its spin limit
    (no timeout elapses) and the kernel returns without writing any output or input."""
    from distributed_torch_horovod_gcp_b200.runtime import symm as S
    N, grid, dtype = 3, 7, BF16
    nvec = 2 * 7 * THREADS * N + 5
    n = nvec * 8
    gen = torch.Generator().manual_seed(5)
    gs = make_grads(N, n, dtype, gen)
    emu, ck = Emu(N, seed=7), Checker()
    inp, out = [_buf(n, dtype, g) for g in gs], [_buf(n, dtype) for _ in range(N)]
    f32 = [_buf(n, F32) for _ in range(N)]
    ints = torch.tensor([0, 0, -7, -7], dtype=torch.int32, device="cuda")
    chunks = torch.tensor([(0, nvec, 0, 1)], dtype=torch.int32, device="cuda")
    lib, st, b = emu.lib, _stream(), ctypes.byref
    r = 1

    def fn(ctx):
        a = ar_args(inp, out, n, 1.0 / N, CH_USER, 1)
        a.step_ctr, a.ticket = ints.data_ptr(), ints.data_ptr() + 4
        if kernel in ("oneshot", "twoshot"):
            return lib.b200dp_comm_allreduce(b(ctx), b(a), 0 if kernel == "oneshot" else 1, 1, grid, THREADS, st)
        if kernel == "clip":
            k = S.ClipArgs()
            k.r, k.slots = f32[0].data_ptr(), f32[1].data_ptr()
            return lib.b200dp_comm_clip_bucket(b(ctx), b(a), b(k), 0, 1, grid, THREADS, st)
        if kernel == "layerwise":
            a.h.kind = S.OPT_LARS
            k = S.LwArgs()
            k.r, k.part, k.chunks, k.nchunks = f32[0].data_ptr(), f32[1].data_ptr(), chunks.data_ptr(), 1
            return lib.b200dp_comm_lw_bucket(b(ctx), b(a), b(k), 0, 1, grid, THREADS, st)
        if kernel == "broadcast":
            c = S.BcastArgs()
            for q in range(N):
                c.buf[q] = out[q].data_ptr()
            c.nbytes, c.root, c.channel = n * 2, r, CH_USER
            return lib.b200dp_comm_broadcast(b(ctx), b(c), grid, THREADS, st)
        c = S.CollArgs()
        for q in range(N):
            c.src[q], c.dst[q] = inp[q].data_ptr(), out[q].data_ptr()
        mode = {"reduce-scatter": 0, "allgather": 1, "alltoall": 2}[kernel]
        c.chunk, c.scale, c.channel = (n // N // 8 * 8 if mode == 0 else nvec // N), 1.0, CH_USER
        return lib.b200dp_comm_collective(b(ctx), b(c), mode, 1, grid, THREADS, st)

    before = [t.clone() for t in inp + out + f32 + [ints]]
    box = emu.box
    box[0] = 1
    try:
        emu.launch(ck, f"watchdog {kernel}", r, fn, CH_USER, grid, uncredited=2)
    finally:
        for i in range(4):
            box[i] = 0
    assert list(box[:4]) == [0, 0, 0, 0]
    for t, t0 in zip(inp + out + f32 + [ints], before):
        ck.same_bits(f"watchdog {kernel} writes nothing", t, t0)
    ck.close()


# ============================================================================================ closing barrier
def _host_mapped(nbytes):
    """Zeroed page-locked host memory mapped into the device: (numpy uint8 view, device pointer)."""
    hp, dp = ctypes.c_uint64(0), ctypes.c_uint64(0)
    assert _rt().lib.b200dp_host_mailbox(nbytes, ctypes.byref(hp), ctypes.byref(dp)) == 0
    return np.ctypeslib.as_array((ctypes.c_uint8 * nbytes).from_address(hp.value)), dp.value


@gpu
@pytest.mark.parametrize("kernel", ["oneshot", "oneshot-in-place", "twoshot", "clip"])
def test_input_is_released_after_the_closing_barrier(kernel):
    """Peers read rank r's gradients until they reach the closing barrier, so rank r may zero them (or copy the
    in-place result over them) only after it.  Isolated launches cannot see when a write happens, so here the
    host plays the peers: the signal pads and rank r's input live in host-mapped memory, rank r is credited for
    the opening barrier only, and once every block has arrived at the closing barrier (its +1 shows in every
    peer's pad) the input must still be bit-unchanged.  Then the host credits the closing barrier."""
    from distributed_torch_horovod_gcp_b200.runtime import symm as S
    N, r, grid, dtype = 3, 1, 7, BF16
    n = (2 * 7 * THREADS * N + 5) * 8
    gen = torch.Generator().manual_seed(23)
    gs = make_grads(N, n, dtype, gen)
    lib, (box, dev) = _rt().lib, mailbox()
    pads_h, pads_d = _host_mapped(N * PAD * 4)
    pads = pads_h.view(np.int32).reshape(N, CHANNELS, BLOCKS, RANKS)
    in_h, in_d = _host_mapped(n * 2)
    in_h[:] = gs[r].view(torch.int16).numpy().view(np.uint8)
    orig = in_h.copy()
    epoch = torch.zeros(PAD, dtype=torch.int32, device="cuda")
    ctx = S.CommCtx()
    for q in range(N):
        ctx.sig[q] = pads_d + q * PAD * 4
    ctx.epoch, ctx.err, ctx.timeout_ns, ctx.rank, ctx.world = epoch.data_ptr(), dev, TIMEOUT_NS, r, N
    inp = [_buf(n, dtype, g) for g in gs]
    out = [_buf(n, dtype) for _ in range(N)]
    f32 = [_buf(n, F32), _buf(S.MAX_BLOCKS, F32)]
    ptrs = [t.data_ptr() for t in inp]
    ptrs[r] = in_d
    a = S.ARArgs()
    for q in range(N):
        a.inp[q], a.out[q] = ptrs[q], (in_d if kernel == "oneshot-in-place" and q == r else out[q].data_ptr())
    a.n, a.scale, a.channel, a.zero_input = n, 1.0 / N, CH_USER, int(kernel != "oneshot-in-place")
    if kernel == "oneshot-in-place":
        a.scratch, a.copy_back = out[r].data_ptr(), 1
    peers = [t for t in range(N) if t != r]
    pads[r][CH_USER, :grid, peers] = 1
    if kernel == "clip":
        k = S.ClipArgs()
        k.r, k.slots = f32[0].data_ptr(), f32[1].data_ptr()
        rc = lib.b200dp_comm_clip_bucket(ctypes.byref(ctx), ctypes.byref(a), ctypes.byref(k), 0, 1, grid, THREADS,
                                         _stream())
    else:
        rc = lib.b200dp_comm_allreduce(ctypes.byref(ctx), ctypes.byref(a), int(kernel == "twoshot"), 1, grid,
                                       THREADS, _stream())
    assert rc == 0, lib.b200dp_comm_last_error()
    t0 = time.monotonic()
    while not all((pads[t][CH_USER, :grid, r] == 2).all() for t in peers) and time.monotonic() - t0 < 10:
        time.sleep(1e-4)
    arrived = all((pads[t][CH_USER, :grid, r] == 2).all() for t in peers)
    unchanged = np.array_equal(in_h, orig)
    pads[r][CH_USER, :grid, peers] = 2
    torch.cuda.synchronize()
    mail = list(box[:4])
    for i in range(4):
        box[i] = 0
    assert arrived and mail == [0, 0, 0, 0], f"closing barrier not reached (mailbox {mail})"
    assert unchanged, f"{kernel}: rank {r}'s input changed before the closing barrier"
    got = torch.from_numpy(in_h.copy()).view(torch.int16)
    want = ref_exact(gs, fp32(1.0 / N), dtype).view(torch.int16) if kernel == "oneshot-in-place" else \
        torch.zeros(n, dtype=torch.int16)
    assert torch.equal(torch.isnan(got.view(dtype)), torch.isnan(want.view(dtype)))
    assert same_values(got.view(dtype), want.view(dtype)), f"{kernel}: input not released after the barrier"


# ============================================================================================ the references (CPU)
def emulate(gs, sigma, dtype, fault=None):
    """The all-reduce in CPU fp32 with an optional fault: a bf16 accumulator, a dropped rank, the reversed rank
    order, or a per-rank pre-scale."""
    f = torch.float32
    order = list(range(len(gs)))
    if fault == "reversed rank order":
        order = order[::-1]
    if fault == "dropped rank":
        order = order[1:]
    acc = torch.zeros(gs[0].shape, dtype=f)
    s = torch.tensor(sigma, dtype=f)
    for q in order:
        if fault == "per-rank pre-scale":
            acc = acc + gs[q].float() * s
        else:
            acc = acc + gs[q].float()
        if fault == "bf16 accumulator":
            acc = acc.to(torch.bfloat16).float()
    return (acc if fault == "per-rank pre-scale" else acc * s).to(dtype)


CPU_CASES = [(N, d, sk) for N in (2, 3, 5, 7, 8) for d in (F32, BF16, F16) for sk in ("one", "inv", "predivide")]


@pytest.mark.parametrize("N,dtype,skind", CPU_CASES)
def test_cpu_reference_within_bound(N, dtype, skind):
    """Reference (1) lies within bound (2) on every value class, subnormals, +-0, NaN and infinities included."""
    gen = torch.Generator().manual_seed(N)
    gs = make_grads(N, 4000, dtype, gen)
    st = fp32(scale_of(skind, N))
    ck = Checker()
    check_sum(ck, f"cpu reference {str(dtype)[6:]}", ref_exact(gs, st, dtype), gs, st, scale_of(skind, N), dtype)
    ck.close()


def test_cpu_fp16_near_max_stays_finite():
    gen = torch.Generator().manual_seed(3)
    gs = make_grads(8, 4000, F16, gen, "fp16max")
    out = ref_exact(gs, fp32(1 / 8), F16)
    assert bool(torch.isfinite(out).all())
    ck = Checker()
    check_sum(ck, "cpu reference f16 near max", out, gs, fp32(1 / 8), 1 / 8, F16)
    ck.close()


@pytest.mark.parametrize("dtype", [F32, BF16])
def test_cpu_tightest_element_beyond_bound_fails(dtype):
    """The element closest to its bound, moved to 1.01x the bound (in float64), fails; at 0.99x it passes."""
    gen = torch.Generator().manual_seed(11)
    N, n = 7, 4000
    gs = [torch.randn(n, generator=gen, dtype=torch.float64).to(dtype) for _ in range(N)]
    sigma = fp32(1 / N)
    out = ref_exact(gs, sigma, dtype).double()
    ideal, _, bound = sum_bound(gs, sigma, 1 / N, dtype)
    ratio = Checker().bound("cpu tightness probe", out, Ev(ideal, bound))
    i = int(torch.argmax(ratio))
    assert 0 < float(ratio[i]) <= 1
    for f, ok in ((1.01, False), (0.99, True)):
        moved = out.clone()
        moved[i] = ideal[i] + f * bound[i]
        ck = Checker()
        ck.bound("cpu tightness probe", moved, Ev(ideal, bound))
        assert (not ck.fails) == ok
    fp64_bounds._WORST.pop("cpu tightness probe", None)


FAULTS = [
    # fault, dtype, world, scale, the checks that must catch it
    ("bf16 accumulator", BF16, 8, "inv", ("rank order", "fp64")),
    ("bf16 accumulator", F32, 4, "one", ("rank order", "fp64")),
    ("dropped rank", BF16, 3, "inv", ("rank order", "fp64")),
    ("reversed rank order", F32, 5, "inv", ("rank order",)),
    ("per-rank pre-scale", F32, 7, "inv", ("rank order",)),
]


@pytest.mark.parametrize("fault,dtype,N,skind,groups", FAULTS, ids=[f"{f[0]}-{str(f[1])[6:]}" for f in FAULTS])
def test_cpu_fault_is_caught(fault, dtype, N, skind, groups):
    """Each fault, in a CPU emulation of the kernel, fails reference (1), bound (2) or both, as listed."""
    gen = torch.Generator().manual_seed(17)
    gs = make_grads(N, 4000, dtype, gen)
    st = fp32(scale_of(skind, N))
    worst = dict(fp64_bounds._WORST)
    ck = Checker()
    check_sum(ck, "cpu fault", emulate(gs, st, dtype, fault), gs, st, scale_of(skind, N), dtype)
    fp64_bounds._WORST.clear()
    fp64_bounds._WORST.update(worst)
    for g in groups:
        assert any(f.startswith(f"cpu fault {g}:") for f in ck.fails), ck.fails or "nothing failed"


def test_cpu_emulation_without_fault_passes():
    gen = torch.Generator().manual_seed(17)
    gs = make_grads(5, 4000, BF16, gen)
    ck = Checker()
    check_sum(ck, "cpu emulation", emulate(gs, fp32(1 / 5), BF16), gs, fp32(1 / 5), 1 / 5, BF16)
    ck.close()
