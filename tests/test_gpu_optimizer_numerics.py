"""Fused optimizer kernel numerics against float64, element by element and one step at a time: the K7 update
epilogue (csrc/comm_kernels.cu ``make_step`` / ``epilogue`` / ``finish_step``) behind the one-shot all-reduce K1, the
clip-by-global-norm kernels K1c / K8 / K9, and the LARS / LAMB kernels K10 / K11.

The C entry points are called directly at world size 1 (``b200dp_comm_allreduce``, ``b200dp_comm_clip_bucket``,
``b200dp_comm_clip_finalize``, ``b200dp_comm_lw_bucket``) with hand-built argument blocks and an explicit grid, so
the grid-stride loops and the last-block step-counter ticket run with one CTA, with 7 and with 128.  Every buffer
has a guard region of NaN past ``n`` that must stay bit-unchanged, and every output the kernel must write starts as
NaN.  A last test drives the same kernels through ``hvd.DistributedOptimizer`` (``B200DP_FUSED_SINGLE=1``) to cover
the engine's hyperparameter plumbing, master copies and per-group buckets.

Each step is checked against float64 computed from the exact values the kernel saw at that step (gradient, master
or fp32 parameter, S0 / S1, step counter), so multi-step runs do not pile up error.  The hyperparameters are the
fp32 values in ``OptHyper``, and ``lr * lr_scale`` is rounded as the kernel rounds it.  The gap between those fp32
hyperparameters and the Python doubles a user writes (for beta2 = 0.999 it moves the update by about
|delta beta| / (1 - beta) = 1.3e-5) is a property of the fp32 argument block, not of the kernels, and is out of
scope here.

Bounds are derived, not fitted.  ``Ev`` carries a float64 value and a bound on the distance to what the kernel
holds.  Every fp32 rounding adds u (|value| + bound) plus 2^-149 absolute (a subnormal result), u = 2^-24, so an fma
counts as a product and a sum rounded separately: that bounds the fused and the unfused form alike, whatever the
compiler contracts.  A result whose whole interval lies past the fp32 overflow threshold is +-inf exactly, as in the
kernel.  With the step counter t, the kernel forms the bias corrections 1 - beta1^t and sqrt(1 - beta2^t) in double
and rounds each to fp32 once; their bound is a few double roundings plus that one fp32 rounding, so an fp32
``1 - powf(beta, t)``, which cancels for beta near 1 and small t, fails the early-step cases.

The reference follows the kernel's operation order.  For Adam's second moment that is ((1 - beta2) g) g, which
overflows later than torch's g * g: a gradient of 1e20 gives v = inf for beta2 = 0.95 in both, a finite v in the
kernel for beta2 >= 0.999.  Squares of gradients near 1e-30 underflow to zero in both.
"""
import ctypes
import math

import numpy as np
import pytest
import torch

import fp64_bounds
from fp64_bounds import U32, report_ratios

gpu = pytest.mark.gpu

TINY = 2.0 ** -149                         # absolute error of a subnormal fp32 result
OVF = 2.0 ** 128 * (1 - 2.0 ** -25)        # |x| at or above this rounds to inf in fp32
U64 = 2.0 ** -53
GUARD = 64                                 # guard elements past n in every buffer
THREADS = 512
LW_CHUNK_ELEMS = 16384                     # as parallel/fused_engine.py
DT_CODE = {torch.float32: 0, torch.bfloat16: 1, torch.float16: 2}
VN = {torch.float32: 4, torch.bfloat16: 8, torch.float16: 8}


@pytest.fixture(scope="module", autouse=True)
def _report_ratios():
    yield
    report_ratios()


# ============================================================================================ error propagation
class Ev:
    """float64 value ``v`` and a bound ``e`` on |kernel value - v| (tensors, broadcastable)."""
    __slots__ = ("v", "e")

    def __init__(self, v, e=None):
        self.v = v
        self.e = torch.zeros_like(v) if e is None else e

    def __neg__(self):
        return Ev(-self.v, self.e)


def _mul0(x, y):
    """x * y with 0 * inf = 0: a bound term that is zero stays zero next to an infinite value."""
    return torch.where((x == 0) | (y == 0), torch.zeros_like(x * y), x * y)


def const(x, like):
    """An exact fp32 scalar or tensor (a hyperparameter read from OptHyper, or values computed bit-exactly)."""
    if torch.is_tensor(x):
        return Ev(x.double().to(like.v.device))
    return Ev(torch.tensor(float(x), dtype=torch.float64, device=like.v.device))


def rnd(x):
    """One fp32 rounding: + u (|v| + e) + 2^-149.  An infinite value, or one whose interval lies wholly at or past
    the overflow threshold, is +-inf exactly; one whose interval straddles the threshold is a choice of data the
    test cannot decide, and raises."""
    mag = x.v.abs() + x.e
    over = torch.isinf(x.v) | ((x.v.abs() - x.e) >= OVF)
    if bool(((mag >= OVF) & ~over).any()):
        raise ValueError("a value within its bound of the fp32 overflow threshold: choose other data")
    v = torch.where(over, torch.sign(x.v) * math.inf, x.v)
    e = torch.where(over, torch.zeros_like(x.e), x.e + U32 * mag + TINY)
    return Ev(v, e)


def add(a, b):
    return rnd(Ev(a.v + b.v, a.e + b.e))


def mul(a, b):
    """|a'b' - ab| <= |a| e_b + |b| e_a + e_a e_b, then one rounding."""
    e = _mul0(a.v.abs(), b.e) + _mul0(b.v.abs(), a.e) + a.e * b.e
    return rnd(Ev(a.v * b.v, e))


def fma(a, b, c):
    """fmaf(a, b, c) or a * b + c: bounded as a rounded product and a rounded sum, which covers both."""
    return add(mul(a, b), c)


def div(a, b):
    """|a'/b' - a/b| <= (|a| e_b + |b| e_a) / (|b| (|b| - e_b)) for |b| > e_b; 0 when b is exactly inf."""
    bb = b.v.abs()
    if bool((bb <= b.e).any()):
        raise ValueError("divisor interval contains 0")
    e = (_mul0(a.v.abs(), b.e) + bb * a.e) / (bb * (bb - b.e))
    e = torch.where(torch.isinf(b.v) & (b.e == 0), torch.zeros_like(e), e)
    return rnd(Ev(a.v / b.v, e))


def sqrt_(a, fp32=True):
    """|sqrt(a') - sqrt(a)| <= min(sqrt(e_a), e_a / sqrt(a)), then one rounding (fp32, or double when not)."""
    r = torch.sqrt(a.v)
    e = torch.sqrt(a.e)
    e = torch.where(r > 0, torch.minimum(e, a.e / r.clamp_min(1e-300)), e)
    e = torch.where(torch.isinf(r) & (a.e == 0), torch.zeros_like(e), e)
    out = Ev(r, e)
    return rnd(out) if fp32 else Ev(r, e + 2 * U64 * r)


def bias_corrections(beta1, beta2, t, dev):
    """(1 - beta1^t, sqrt(1 - beta2^t)) as Ev, t >= 1, the kernel's ``bias_corrections``: the double ``pow`` is
    within 2 ulp (CUDA C Programming Guide), 2^-51 beta^t, and so is this reference's own pow; ``1 - pow`` rounds
    once in double, 2^-53 (1 - beta^t); the double sqrt rounds once more; each factor is rounded to fp32 once."""
    def w(beta):
        bt = float(beta) ** t
        return Ev(torch.tensor(1.0 - bt, dtype=torch.float64, device=dev),
                  torch.tensor(2 * 2.0 ** -51 * bt + 2 * U64 * (1.0 - bt), dtype=torch.float64, device=dev))
    return rnd(w(beta1)), rnd(sqrt_(w(beta2), fp32=False))


# ============================================================================================ update references
def k7_ref(g, p, s0, s1, h, t, lr, scale):
    """The K7 epilogue in float64 with bounds, from the exact inputs of one launch.

    g: the gradient the kernel read (float64 of the bucket dtype), p: master (or fp32 parameter), s0 / s1: the
    state before the launch, h: OptHyper as a dict of fp32 values, t: the step counter before the launch, lr: the
    kernel's fp32 ``h.lr * lr_scale`` (exact), scale: ARArgs.scale.  Returns {"p", "s0", "s1"} of the state the
    kernel writes (a key is missing when the kernel must not write that buffer).  Operation order as the kernel:
    - g = fl(g * scale) (exact when scale == 1), negated for ``maximize``;
    - SGD: g = fma(wd, p, g) when wd != 0; with momentum, b = g on the first step (t == 0), else
      b = fma(momentum, s0, fl(1 - dampening) g); g = nesterov ? fma(momentum, b, g) : b; p = fma(-lr, g, p);
    - Adam: AdamW scales p by fl(1 - fl(lr wd)), Adam adds fma(wd, p, g); m = fma(b1, m, fl(1 - b1) g);
      v = fma(b2, v, fl(1 - b2) g g); p = fma(-(lr / bc1), m / (sqrt(v) / bc2 + eps), p)."""
    dev = g.device
    G, P = Ev(g), Ev(p)
    c = lambda x: const(x, G)   # noqa: E731
    if scale != 1.0:
        G = mul(G, c(scale))
    if h["maximize"]:
        G = -G
    out = {}
    if h["kind"] == 1:
        if h["weight_decay"] != 0.0:
            G = fma(c(h["weight_decay"]), P, G)
        if h["momentum"] != 0.0:
            if t == 0:
                B = G
            else:
                B = fma(c(h["momentum"]), Ev(s0), mul(rnd(add(c(1.0), -c(h["dampening"]))), G))
            out["s0"] = B
            G = fma(c(h["momentum"]), B, G) if h["nesterov"] else B
        out["p"] = fma(-c(lr), G, P)
        return out
    bc1, bc2 = bias_corrections(h["beta1"], h["beta2"], t + 1, dev)
    if h["adamw"]:
        P = mul(P, add(c(1.0), -mul(c(lr), c(h["weight_decay"]))))
    elif h["weight_decay"] != 0.0:
        G = fma(c(h["weight_decay"]), P, G)
    M = fma(c(h["beta1"]), Ev(s0), mul(add(c(1.0), -c(h["beta1"])), G))
    V = fma(c(h["beta2"]), Ev(s1), mul(mul(add(c(1.0), -c(h["beta2"])), G), G))
    den = add(div(sqrt_(V), bc2), c(h["eps"]))
    out["p"] = fma(-div(c(lr), bc1), div(M, den), P)
    out["s0"], out["s1"] = M, V
    return out


def lamb_dir_ref(g, p, s0, s1, h, t, scale):
    """K10's LAMB update direction and moments: g = fl(g * scale); m = fma(b1, m, fl(1 - b1) g);
    v = fma(b2, v, fl(1 - b2) g g); r = fma(wd, p, (m / bc1) / (sqrt(v) / bc2 + eps)).  LARS (h kind 3):
    r = fma(wd, p, g), no state."""
    G, P = Ev(g), Ev(p)
    c = lambda x: const(x, G)   # noqa: E731
    if scale != 1.0:
        G = mul(G, c(scale))
    if h["kind"] == 3:
        return {"r": fma(c(h["weight_decay"]), P, G)}
    bc1, bc2 = bias_corrections(h["beta1"], h["beta2"], t + 1, g.device)
    M = fma(c(h["beta1"]), Ev(s0), mul(add(c(1.0), -c(h["beta1"])), G))
    V = fma(c(h["beta2"]), Ev(s1), mul(mul(add(c(1.0), -c(h["beta2"])), G), G))
    den = add(div(sqrt_(V), bc2), c(h["eps"]))
    return {"r": fma(c(h["weight_decay"]), P, div(div(M, bc1), den)), "s0": M, "s1": V}


def lw_apply_ref(r, p, s0, h, step):
    """K11 from the kernel's direction r and the exact fp32 ``step = lr * trust``: LAMB p = fma(-step, r, p);
    LARS b = fma(momentum, b, fl(step r)), p = fl(p - b)."""
    R, P = Ev(r), Ev(p)
    c = lambda x: const(x, R)   # noqa: E731
    if h["kind"] == 4:
        return {"p": fma(-c(step), R, P)}
    B = fma(c(h["momentum"]), Ev(s0), mul(c(step), R))
    return {"p": add(P, -B), "s0": B}


# ============================================================================================ checking
class Checker:
    """Collects every group that fails, so a test (and the fault checks below) can see which groups caught it."""

    def __init__(self):
        self.fails = []

    def bound(self, group, out, ref):
        out64 = out.detach().double()
        v, e = torch.broadcast_to(ref.v, out64.shape), torch.broadcast_to(ref.e, out64.shape)
        same = out64 == v                                    # equal values, equal infinities included
        err = torch.where(same, torch.zeros_like(out64), (out64 - v).abs())
        ratio = torch.where(e > 0, err / e.clamp_min(1e-300),
                            torch.where(err > 0, torch.full_like(err, math.inf), torch.zeros_like(err)))
        ratio = torch.where(torch.isnan(ratio), torch.full_like(ratio, math.inf), ratio)
        worst = int(torch.argmax(ratio)) if ratio.numel() else 0
        r = float(ratio.reshape(-1)[worst]) if ratio.numel() else 0.0
        fp64_bounds._WORST[group] = max(fp64_bounds._WORST.get(group, 0.0), r)
        if not r <= 1.0:
            self.fails.append(f"{group}: {int((ratio > 1).sum())} element(s) outside the bound; worst at {worst}: "
                              f"out={float(out64.reshape(-1)[worst]):.9g} ref={float(v.reshape(-1)[worst]):.9g} "
                              f"err/bound={r:.3g}")
        return ratio

    def true(self, group, ok, what=""):
        if not ok:
            self.fails.append(f"{group}: {what}")

    def same_bits(self, group, a, b):
        self.true(group, torch.equal(_bits(a), _bits(b)), "bits differ")

    def close(self):
        if self.fails:
            raise AssertionError("\n".join(self.fails))


def _bits(t):
    return t.contiguous().view({4: torch.int32, 2: torch.int16}[t.element_size()])


def _f32(x):
    return float(np.float32(x))


# ============================================================================================ direct kernel calls
def _rt():
    from distributed_torch_horovod_gcp_b200.runtime.local import LocalRuntime
    rt = LocalRuntime.get()
    assert rt is not None, "native comm library not loaded"
    return rt


def _buf(n, dtype, data=None):
    t = torch.full((n + GUARD,), math.nan, dtype=dtype, device="cuda")
    if data is not None:
        t[:n] = data
    return t


HYPER_FIELDS = ("kind", "nesterov", "adamw", "maximize", "lr", "momentum", "dampening", "weight_decay",
                "beta1", "beta2", "eps")


class DirectBucket:
    """One bucket's buffers for direct kernel calls: gradient ``g``, output ``out``, fp32 master ``M`` (16-bit
    dtypes), state ``S0`` / ``S1`` and ``ints`` = [step counter, ticket, sentinels].  Each has GUARD NaN (or
    sentinel) elements past n."""

    def __init__(self, dtype, n, p, s0=None, s1=None, t=0, lr_scale=None):
        self.dtype, self.n = dtype, n
        self.g = _buf(n, dtype, 0.0)
        if dtype == torch.float32:
            self.M, self.out = None, _buf(n, torch.float32, p)
        else:
            self.M, self.out = _buf(n, torch.float32, p), _buf(n, dtype)
        self.S0 = _buf(n, torch.float32, s0)
        self.S1 = _buf(n, torch.float32, s1)
        self.ints = torch.tensor([t, 0, -7, -7, -7, -7, -7, -7], dtype=torch.int32, device="cuda")
        self.lr_scale = None if lr_scale is None else torch.tensor([lr_scale, math.nan], device="cuda")

    def master(self):
        return self.M if self.M is not None else self.out

    def args(self, hyper, scale, s1=True):
        from distributed_torch_horovod_gcp_b200.runtime import symm as S
        a = S.ARArgs()
        a.inp[0], a.out[0] = self.g.data_ptr(), self.out.data_ptr()
        a.master = self.M.data_ptr() if self.M is not None else 0
        a.s0 = self.S0.data_ptr()
        a.s1 = self.S1.data_ptr() if s1 else 0
        a.step_ctr, a.ticket = self.ints.data_ptr(), self.ints.data_ptr() + 4
        a.lr_scale = self.lr_scale.data_ptr() if self.lr_scale is not None else 0
        a.n, a.scale, a.channel, a.zero_input, a.copy_back = self.n, scale, S.CH_USER, 1, 0
        for k, v in hyper.items():
            setattr(a.h, k, v)
        h = {k: getattr(a.h, k) for k in HYPER_FIELDS}            # the fp32 values the kernel reads
        lr = _f32(np.float32(h["lr"]) * np.float32(float(self.lr_scale[0]))) if self.lr_scale is not None \
            else h["lr"]
        return a, h, lr, float(a.scale)

    def snapshot(self):
        n = self.n
        bufs = {k: getattr(self, k) for k in ("g", "out", "M", "S0", "S1") if getattr(self, k) is not None}
        return {"in": {k: b[:n].clone() for k, b in bufs.items()}, "guard": {k: b[n:].clone() for k, b in bufs.items()},
                "t": int(self.ints[0])}

    def check_common(self, ck, snap, tag, k7_written):
        """Guards bit-unchanged, gradient zeroed over [0, n), counter +1 and ticket back at 0, output = RN(master)."""
        n = self.n
        for k, gb in snap["guard"].items():
            ck.same_bits(f"{tag} guard", getattr(self, k)[n:], gb)
        ck.true(f"{tag} zero_input", bool((self.g[:n] == 0).all()), "gradient not zeroed")
        ints = self.ints.tolist()
        ck.true(f"{tag} step counter", ints[0] == snap["t"] + 1 and ints[1] == 0 and ints[2:] == [-7] * 6,
                f"ints {ints} after step counter {snap['t']}")
        if self.M is not None:
            ck.same_bits(f"{tag} {str(self.dtype)[6:]} store", self.out[:n], self.M[:n].to(self.dtype))
        for k in ("S0", "S1"):
            if k not in k7_written:
                ck.same_bits(f"{tag} {k} untouched", getattr(self, k)[:n], snap["in"][k])


def _launch_allreduce(bk, a, blocks):
    rt = _rt()
    rc = rt.lib.b200dp_comm_allreduce(ctypes.byref(rt.ctx), ctypes.byref(a), 0, DT_CODE[bk.dtype], blocks, THREADS,
                                      torch.cuda.current_stream().cuda_stream)
    assert rc == 0, rt.lib.b200dp_comm_last_error()


def check_k7(ck, bk, snap, h, lr, scale, tag, g_seen=None):
    """Everything one K7 (or K9, with ``g_seen`` = fl(r coef) and scale 1) launch wrote, against float64."""
    n = bk.n
    g = snap["in"]["g"].double() if g_seen is None else g_seen.double()
    p0 = snap["in"]["M" if bk.M is not None else "out"].double()
    ref = k7_ref(g, p0, snap["in"]["S0"].double(), snap["in"]["S1"].double(), h, snap["t"], lr, scale)
    ck.bound(f"{tag} master", bk.master()[:n], ref["p"])
    for k in ("s0", "s1"):
        if k in ref:
            ck.bound(f"{tag} {k.upper()}", getattr(bk, k.upper())[:n], ref[k])
    bk.check_common(ck, snap, tag, {k.upper() for k in ref if k != "p"})


def _nvec(kind, blocks, vn):
    return {"one": 1, "small": 37, "sweep": blocks * THREADS + 37}[kind] * vn


def _grads(n, dtype, gen, wide=True):
    """Normal gradients, with every third element log-uniform over 1e-30 .. 1e20 (1e-7 .. 6e4 for fp16)."""
    g = torch.randn(n, generator=gen, dtype=torch.float64)
    if wide:
        lo, hi = (-7.0, 4.7) if dtype == torch.float16 else (-30.0, 20.0)
        k = torch.arange(0, n, 3)
        e = lo + (hi - lo) * torch.rand(k.numel(), generator=gen, dtype=torch.float64)
        g[k] = torch.sign(g[k]) * 10.0 ** e
    return g.to(dtype).cuda()


def _state(n, gen, t, adam):
    p = torch.randn(n, generator=gen).cuda()
    if t == 0 and adam:
        return p, torch.zeros(n, device="cuda"), torch.zeros(n, device="cuda")
    s0 = (0.1 * torch.randn(n, generator=gen)).cuda()
    s1 = (0.01 * torch.randn(n, generator=gen) ** 2).cuda()
    return p, s0, s1


def run_k7(dtype, blocks, n, hyper, t, scale, lr_scale, steps=1, seed=0, tag=None, wide=True):
    """Launch K1 + K7 ``steps`` times from step counter t, each step checked from the kernel's own state."""
    gen = torch.Generator().manual_seed(seed)
    adam = hyper["kind"] == 2
    p, s0, s1 = _state(n, gen, t, adam)
    if not adam and t == 0:
        s0 = None                        # the first SGD step must not read S0: NaN there would show
    bk = DirectBucket(dtype, n, p, s0, s1 if adam else torch.randn(n, generator=gen).cuda(), t, lr_scale)
    tag = tag or ("sgd" if not adam else ("adamw" if hyper.get("adamw") else "adam"))
    for _ in range(steps):
        bk.g[:n] = _grads(n, dtype, gen, wide)
        if bk.M is not None:
            bk.out[:n] = math.nan
        a, h, lr, sc = bk.args(hyper, scale, s1=adam)
        snap = bk.snapshot()
        _launch_allreduce(bk, a, blocks)
        torch.cuda.synchronize()
        ck = Checker()
        check_k7(ck, bk, snap, h, lr, sc, tag)
        ck.close()
    return bk


SGD = dict(kind=1)
ADAM = dict(kind=2, beta1=0.9, beta2=0.999, eps=1e-8)
F32, BF16, F16 = torch.float32, torch.bfloat16, torch.float16

SGD_CASES = [
    # id, dtype, blocks, size, scale, hyperparameters, step counter, lr_scale
    ("first-f32-1cta", F32, 1, "one", 1.0, dict(lr=0.5, momentum=0.9, dampening=0.3, weight_decay=1e-2), 0, None),
    ("first-f16-damp", F16, 1, "sweep", 1 / 8, dict(lr=0.5, momentum=0.9, dampening=0.3), 0, None),
    ("later-damp-bf16", BF16, 7, "sweep", 1 / 8, dict(lr=0.5, momentum=0.9, dampening=0.3, weight_decay=1e-2), 5,
     None),
    ("nesterov-f16-128cta", F16, 128, "sweep", 3 / 8, dict(lr=0.25, momentum=0.9, nesterov=1, weight_decay=1e-4), 3,
     0.5),
    ("mom0-max-bf16", BF16, 7, "small", 1.0, dict(lr=0.5, momentum=0.0, weight_decay=0.1, maximize=1), 2, None),
    ("mom0-f32-128cta", F32, 128, "sweep", 1 / 8, dict(lr=0.5), 0, 0.25),
    ("max-nesterov-f32", F32, 7, "sweep", 3 / 8, dict(lr=0.5, momentum=0.9, nesterov=1, maximize=1,
                                                      weight_decay=1e-2), 7, None),
    ("lrscale-bf16-128cta", BF16, 128, "sweep", 1.0, dict(lr=0.5, momentum=0.9, dampening=0.3), 1, 0.3),
]


@gpu
@pytest.mark.parametrize("case", SGD_CASES, ids=[c[0] for c in SGD_CASES])
def test_sgd_step(case):
    _, dtype, blocks, size, scale, hyper, t, lr_scale = case
    run_k7(dtype, blocks, _nvec(size, blocks, VN[dtype]), dict(SGD, **hyper), t, scale, lr_scale)


ADAM_CASES = [
    ("f32-1cta-one", F32, 1, "one", 1.0, dict(lr=0.5), 0, None),
    ("bf16-7cta-l2", BF16, 7, "sweep", 1 / 8, dict(lr=0.5, weight_decay=1e-2), 4, None),
    ("f16-128cta-max", F16, 128, "sweep", 3 / 8, dict(lr=0.25, maximize=1, eps=1e-3), 9, 0.5),
    ("f32-7cta-adamw-lrscale", F32, 7, "sweep", 1.0, dict(lr=0.5, adamw=1, weight_decay=0.1), 2, 0.3),
    ("bf16-1cta-adamw-max", BF16, 1, "sweep", 1 / 8, dict(lr=0.5, adamw=1, weight_decay=0.1, maximize=1,
                                                           beta2=0.95), 0, None),
    ("f16-7cta-adamw-eps", F16, 7, "small", 1.0, dict(lr=0.5, adamw=1, weight_decay=1e-2, eps=1e-3,
                                                       beta2=0.9999), 1, 0.25),
    ("f32-128cta-l2-max", F32, 128, "sweep", 3 / 8, dict(lr=0.5, weight_decay=0.1, maximize=1, beta2=0.99999), 26,
     None),
]


@gpu
@pytest.mark.parametrize("case", ADAM_CASES, ids=[c[0] for c in ADAM_CASES])
def test_adam_step(case):
    _, dtype, blocks, size, scale, hyper, t, lr_scale = case
    run_k7(dtype, blocks, _nvec(size, blocks, VN[dtype]), dict(ADAM, **hyper), t, scale, lr_scale)


@gpu
@pytest.mark.parametrize("beta2", [0.95, 0.999, 0.9999, 0.99999])
@pytest.mark.parametrize("t", [1, 2, 3, 10, 27, 10 ** 3, 10 ** 6])
def test_adam_bias_correction(beta2, t):
    """Step t (counter t - 1) with the tight bias-correction bound.  lr = 0.5 and unit-sized moments make the
    update as large as the parameter, so an fp32 1 - beta2^t (tens to thousands of u for beta2 >= 0.999 at small
    t) shows in the master."""
    run_k7(F32, 7, 3000 * 4, dict(ADAM, lr=0.5, beta2=beta2), t - 1, 1.0, None, wide=False, seed=t)


@gpu
@pytest.mark.parametrize("dtype", [F32, BF16, F16])
@pytest.mark.parametrize("kind", ["sgd", "adam"])
def test_multi_step(dtype, kind):
    """20 steps from a zero counter, each from the state the previous launch left."""
    hyper = dict(SGD, lr=0.5, momentum=0.9, dampening=0.3, weight_decay=1e-2) if kind == "sgd" else \
        dict(ADAM, lr=0.5, weight_decay=1e-2, beta2=0.9999)
    bk = run_k7(dtype, 7, _nvec("sweep", 7, VN[dtype]), hyper, 0, 1 / 8, None, steps=20, seed=3)
    assert int(bk.ints[0]) == 20


@gpu
def test_fp16_store_overflows_while_master_stays_finite():
    """Masters past 65504 round to inf in the fp16 output (as ``master.to(float16)``), and stay finite."""
    bk = run_k7(F16, 7, _nvec("small", 7, 8), dict(SGD, lr=4.0), 1, 1.0, None, tag="sgd f16 overflow")
    n = bk.n
    assert bool(torch.isinf(bk.out[:n]).any()) and bool(torch.isfinite(bk.M[:n]).all())


@gpu
@pytest.mark.parametrize("t0", [10 ** 3, 10 ** 6])
def test_adam_late_steps(t0):
    run_k7(BF16, 7, _nvec("small", 7, 8), dict(ADAM, lr=0.5, adamw=1, weight_decay=0.1), t0, 1.0, 0.5, steps=3)


# -------------------------------------------------------------------------------------------- clip: K1c / K8 / K9
@gpu
@pytest.mark.parametrize("dtype,blocks,max_norm,kind", [
    (F32, 7, 1e-3, "adam"), (BF16, 128, 1e30, "sgd"), (F16, 1, 1e-2, "sgd"), (BF16, 7, 0.5, "adam")])
def test_clip_kernels(dtype, blocks, max_norm, kind):
    from distributed_torch_horovod_gcp_b200.runtime import symm as S
    rt = _rt()
    vn = VN[dtype]
    n = _nvec("sweep", blocks, vn) + 3 * blocks * THREADS * vn       # several sweeps plus a partial one
    gen = torch.Generator().manual_seed(7)
    adam = kind == "adam"
    hyper = dict(ADAM, lr=0.5, weight_decay=1e-2) if adam else dict(SGD, lr=0.5, momentum=0.9, dampening=0.3)
    p, s0, s1 = _state(n, gen, 2, adam)
    bk = DirectBucket(dtype, n, p, s0, s1, 2)
    bk.g[:n] = _grads(n, dtype, gen, wide=False)
    r = _buf(n, torch.float32)
    slots = torch.zeros(S.MAX_BLOCKS + GUARD, device="cuda")
    slots[:blocks] = math.nan
    slots[S.MAX_BLOCKS:] = math.nan
    scal = torch.full((8,), math.nan, device="cuda")          # norm, coef, guard
    k = S.ClipArgs()
    k.r, k.slots, k.norm, k.coef = r.data_ptr(), slots.data_ptr(), scal.data_ptr(), scal.data_ptr() + 4
    k.max_norm, k.nslots = max_norm, S.MAX_BLOCKS
    scale = 1 / 8
    a, h, lr, sc = bk.args(hyper, scale, s1=adam)
    snap = bk.snapshot()
    st = torch.cuda.current_stream().cuda_stream
    assert rt.lib.b200dp_comm_clip_bucket(ctypes.byref(rt.ctx), ctypes.byref(a), ctypes.byref(k), 0,
                                          DT_CODE[dtype], blocks, THREADS, st) == 0
    assert rt.lib.b200dp_comm_clip_finalize(ctypes.byref(k), st) == 0
    ap = S.ARArgs.from_buffer_copy(a)
    ap.scale = 1.0
    assert rt.lib.b200dp_comm_clip_bucket(ctypes.byref(rt.ctx), ctypes.byref(ap), ctypes.byref(k), 1,
                                          DT_CODE[dtype], blocks, THREADS, st) == 0
    torch.cuda.synchronize()
    ck = Checker()
    # K1c: r = fl(scale g), bit for bit; the guard stays NaN
    ck.true("clip r", torch.equal(r[:n], snap["in"]["g"].float() * np.float32(sc)), "r != fl(scale g)")
    ck.same_bits("clip r guard", r[n:], torch.full((GUARD,), math.nan, device="cuda"))
    # K1c slots: CTA b holds the vectors v with (v mod grid) // 512 == b; sequential fma per thread, two 32-wide
    # butterflies and one 16-wide fold: an any-order bound over vn * (vectors per thread) + 10 terms
    nvec = n // vn
    r64 = r[:n].double().reshape(nvec, vn)
    cta = (torch.arange(nvec, device="cuda") % (blocks * THREADS)) // THREADS
    sq = torch.zeros(blocks, dtype=torch.float64, device="cuda").index_add_(0, cta, (r64 * r64).sum(1))
    per_thread = -(-nvec // (blocks * THREADS))
    depth = vn * per_thread + 10
    ck.bound("clip slots", slots[:blocks], Ev(sq, 2 * depth * U32 * sq + depth * THREADS * TINY))
    ck.true("clip slots guard", bool((slots[blocks:S.MAX_BLOCKS] == 0).all()) and
            bool(torch.isnan(slots[S.MAX_BLOCKS:]).all()), "slots past the grid were written")
    # K8: the slots in double, sqrt, one fp32 rounding; coef = min(fl(fl(1 / fl(norm + 1e-6)) max_norm), 1)
    tot = slots[:blocks].double().sum()
    norm = rnd(sqrt_(Ev(tot, S.MAX_BLOCKS * U64 * tot), fp32=False))
    ck.bound("clip norm", scal[0:1], norm)
    nk = np.float32(float(scal[0]))
    coef = min(np.float32(np.float32(1.0) / np.float32(nk + np.float32(1e-6))) * np.float32(max_norm),
               np.float32(1.0))
    ck.true("clip coef", float(scal[1]) == float(coef), f"coef {float(scal[1])!r} != {float(coef)!r}")
    ck.true("clip coef < 1" if max_norm < 1 else "clip coef == 1", (float(coef) < 1.0) == (max_norm < 1))
    ck.same_bits("clip scalars guard", scal[2:], torch.full((6,), math.nan, device="cuda"))
    # K9: the K7 check on fl(r coef)
    check_k7(ck, bk, snap, h, lr, 1.0, f"clip {kind}", g_seen=r[:n] * torch.tensor(coef, device="cuda"))
    ck.close()


# -------------------------------------------------------------------------------------------- LARS / LAMB: K10 / K11
def _lw_layout(dtype, sizes):
    """Tensors at 16-byte boundaries, chunk rows as parallel/fused_engine.py builds them: (first_vec, nvec, tfirst,
    tcount).  Returns (n, [(offset, numel, first chunk)], rows)."""
    vn = VN[dtype]
    per = LW_CHUNK_ELEMS // vn
    rows, tens, off = [], [], 0
    for numel in sizes:
        v0, nv = off // vn, -(-numel // vn)
        cnt = -(-nv // per)
        tens.append((off, numel, len(rows)))
        t0 = len(rows)
        rows += [(v0 + c * per, min(per, nv - c * per), t0, cnt) for c in range(cnt)]
        off += nv * vn
    return off, tens, rows


@gpu
@pytest.mark.parametrize("dtype,kind,adaptive,blocks", [
    (F32, "lamb", True, 7), (BF16, "lamb", True, 128), (F16, "lamb", False, 1),
    (F32, "lars", True, 1), (BF16, "lars", False, 7), (F16, "lars", True, 7)])
def test_layerwise_kernels(dtype, kind, adaptive, blocks):
    """K10 / K11 per element: the direction r, LAMB's moments and the update from the kernel's own trust ratio.
    Tensors: one of 5 chunks + 5 elements (its last vector ends in padding), an all-zero one (ratio 1), and
    small ones, so CTAs walk several chunks each."""
    from distributed_torch_horovod_gcp_b200.runtime import symm as S
    rt = _rt()
    n, tens, rows = _lw_layout(dtype, [5 * LW_CHUNK_ELEMS + 5, 100, 7, 1000, 3 * LW_CHUNK_ELEMS])
    nch = len(rows)
    gen = torch.Generator().manual_seed(11)
    lamb = kind == "lamb"
    t = 4
    p, s0, s1 = _state(n, gen, t, True)
    g = _grads(n, dtype, gen, wide=False)
    live = torch.zeros(n, dtype=torch.bool)
    for off, numel, _ in tens:
        live[off: off + numel] = True
    zero_t = tens[1]
    live_z = live.clone()
    live_z[zero_t[0]: zero_t[0] + zero_t[1]] = False
    live, live_z = live.cuda(), live_z.cuda()
    p, s0, s1 = p * live_z, s0 * live_z, s1 * live_z          # padding and the all-zero tensor are zero everywhere
    g = torch.where(live_z, g, torch.zeros_like(g))
    bk = DirectBucket(dtype, n, p, s0, s1, t, lr_scale=0.5)
    bk.g[:n] = g
    r = _buf(n, torch.float32)
    part = _buf(2 * nch, torch.float32)
    ratio = _buf(nch, torch.float32)
    chunks = torch.tensor(rows, dtype=torch.int32, device="cuda")
    k = S.LwArgs()
    k.r, k.part, k.ratio, k.chunks, k.nchunks = r.data_ptr(), part.data_ptr(), ratio.data_ptr(), chunks.data_ptr(), nch
    k.adaptive, k.trust_coef = int(adaptive), (0.02 if kind == "lars" else 1.0)
    hyper = dict(kind=4, lr=0.25, beta1=0.9, beta2=0.999, eps=1e-6, weight_decay=0.1) if lamb else \
        dict(kind=3, lr=0.5, momentum=0.9, weight_decay=1e-2)
    a, h, lr, sc = bk.args(hyper, 1 / 8, s1=lamb)
    snap = bk.snapshot()
    st = torch.cuda.current_stream().cuda_stream
    for phase in (0, 1):
        assert rt.lib.b200dp_comm_lw_bucket(ctypes.byref(rt.ctx), ctypes.byref(a), ctypes.byref(k), phase,
                                            DT_CODE[dtype], blocks, THREADS, st) == 0
    torch.cuda.synchronize()
    ck = Checker()
    ins = snap["in"]
    d = lamb_dir_ref(ins["g"].double(), ins["M" if bk.M is not None else "out"].double(), ins["S0"].double(),
                     ins["S1"].double(), h, t, sc)
    ck.bound(f"{kind} direction", r[:n], d["r"])
    ck.same_bits(f"{kind} r guard", r[n:], torch.full((GUARD,), math.nan, device="cuda"))
    written = set()
    if lamb:
        ck.bound("lamb S0", bk.S0[:n], d["s0"])
        ck.bound("lamb S1", bk.S1[:n], d["s1"])
        written = {"S0", "S1"}
    # K11 from the kernel's ratio of each tensor (written at its first chunk only) and its r
    rat = ratio[:nch].tolist()
    steps = torch.empty(n, dtype=torch.float64, device="cuda")
    firsts = {f for _, _, f in tens}
    for off, numel, f in tens:
        tr = rat[f]
        ck.true(f"{kind} trust ratio", math.isfinite(tr) and tr > 0, f"ratio {tr}")
        if not adaptive or (off, numel, f) == zero_t:
            ck.true(f"{kind} trust ratio is 1", tr == 1.0, f"tensor at {off}: ratio {tr}")
        nv = -(-numel // VN[dtype])
        steps[off: off + nv * VN[dtype]] = _f32(np.float32(lr) * np.float32(tr))
    ck.true(f"{kind} ratio slots", all(math.isnan(x) for i, x in enumerate(rat) if i not in firsts), "non-first")
    ck.same_bits(f"{kind} ratio guard", ratio[nch:], torch.full((GUARD,), math.nan, device="cuda"))
    ck.true(f"{kind} partials", bool(torch.isfinite(part[:2 * nch]).all()) and bool(torch.isnan(part[2 * nch:]).all()))
    ap = lw_apply_ref(r[:n].double(), ins["M" if bk.M is not None else "out"].double(), ins["S0"].double(), h, steps)
    ck.bound(f"{kind} master", bk.master()[:n], ap["p"])
    if not lamb:
        ck.bound("lars S0", bk.S0[:n], ap["s0"])
        written = {"S0"}
    bk.check_common(ck, snap, kind, written)
    ck.close()


# ============================================================================================ through the engine
@pytest.fixture
def hvd1(monkeypatch):
    monkeypatch.setenv("B200DP_FUSED_SINGLE", "1")
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK", "LOCAL_WORLD_SIZE", "HOROVOD_TIMELINE"):
        monkeypatch.delenv(k, raising=False)
    import distributed_torch_horovod_gcp_b200.torch as hvd
    hvd.shutdown()
    hvd.init()
    yield hvd
    hvd.shutdown()


def _group_hyper(kind, group):
    """What ``FusedEngine._fill_hyper`` should write for a param group, as OptHyper fp32 values."""
    from distributed_torch_horovod_gcp_b200.runtime import symm as S
    hp = S.OptHyper()
    hp.lr, hp.weight_decay, hp.maximize = group["lr"], group["weight_decay"], int(group["maximize"])
    if kind == "sgd":
        hp.kind, hp.momentum, hp.dampening, hp.nesterov = 1, group["momentum"], group["dampening"], group["nesterov"]
    else:
        hp.kind = 2
        hp.beta1, hp.beta2, hp.eps = group["betas"][0], group["betas"][1], group["eps"]
        hp.adamw = int(bool(group.get("decoupled_weight_decay", False)))
    return {k: getattr(hp, k) for k in HYPER_FIELDS}


@gpu
@pytest.mark.parametrize("dtype", [BF16, F16])
@pytest.mark.parametrize("kind", ["sgd", "adam"])
def test_engine_against_float64(hvd1, dtype, kind):
    """``hvd.DistributedOptimizer`` at world size 1: two param groups with different hyperparameters, small
    buckets plus one bucket large enough for several CTAs, ``engine.lr_scale``.  Gradients are written into the
    arena views and ``step()`` launches every bucket; every parameter is checked against float64 from the arena
    state read before the step."""
    from distributed_torch_horovod_gcp_b200.parallel.fused_engine import arena_view
    hvd = hvd1
    torch.manual_seed(0)
    big = torch.nn.Linear(300, 260)                   # 78,000 weights: more than one CTA of its own bucket
    small = torch.nn.Sequential(torch.nn.Linear(13, 37), torch.nn.Linear(37, 5), torch.nn.Linear(5, 3))
    model = torch.nn.ModuleDict({"big": big, "small": small}).cuda().to(dtype)
    if kind == "sgd":
        groups = [{"params": list(small.parameters()), "momentum": 0.9, "dampening": 0.3, "maximize": True,
                   "weight_decay": 1e-2},
                  {"params": list(big.parameters()), "momentum": 0.0, "weight_decay": 0.1, "lr": 0.25}]
        base = torch.optim.SGD(groups, lr=0.5)
    else:
        groups = [{"params": list(small.parameters()), "weight_decay": 1e-2, "maximize": True},
                  {"params": list(big.parameters()), "weight_decay": 0.1, "decoupled_weight_decay": True,
                   "betas": (0.8, 0.9999), "eps": 1e-3, "lr": 0.25}]
        base = torch.optim.Adam(groups, lr=0.5, betas=(0.9, 0.999))
    opt = hvd.DistributedOptimizer(base, named_parameters=model.named_parameters(), bucket_bytes=512)
    eng = opt.fused_engine
    assert eng is not None and eng.kind == kind
    buckets = opt.bucket_plan()
    assert len(buckets) >= 4 and {b.group_index for b in buckets} == {0, 1}
    assert max(eng.symm.pick_blocks(0, b.nbytes) for b in buckets) > 1
    eng.lr_scale = torch.tensor(0.5, device="cuda")
    for ar in eng.arenas.values():                   # masters start as the parameters
        assert torch.equal(ar["M"], ar["p"].float())
    gen = torch.Generator().manual_seed(1)
    for step in range(3):
        with torch.no_grad():
            for p in model.parameters():
                p.grad.copy_(_grads(p.numel(), dtype, gen).reshape(p.shape))
        ar = eng.arenas[dtype]
        snap = {k: ar[k].clone() for k in ("g", "M", "S0", "S1") if ar[k] is not None}
        ctr = eng.step_ctr.clone()
        launches = eng.kernel_launches
        opt.step()
        torch.cuda.synchronize()
        assert eng.kernel_launches == launches + len(buckets)
        assert torch.equal(eng.step_ctr, ctr + 1) and bool((eng.ticket == 0).all())
        ck = Checker()
        for b in buckets:
            lo, hi = b.flat_offset, b.flat_offset + b.numel
            h = _group_hyper(kind, opt.param_groups[b.group_index])
            lr = _f32(np.float32(h["lr"]) * np.float32(0.5))
            s1 = snap["S1"][lo:hi].double() if "S1" in snap else None
            ref = k7_ref(snap["g"][lo:hi].double(), snap["M"][lo:hi].double(), snap["S0"][lo:hi].double(), s1, h,
                         int(ctr[b.index]), lr, 1.0)
            tag = f"engine {kind}"
            ck.bound(f"{tag} master", ar["M"][lo:hi], ref["p"])
            for key in ("s0", "s1"):
                if key in ref:
                    ck.bound(f"{tag} {key.upper()}", ar[key.upper()][lo:hi], ref[key])
            if "s0" not in ref:
                ck.same_bits(f"{tag} S0 untouched", ar["S0"][lo:hi], snap["S0"][lo:hi])
            for s in b.slots:
                ck.same_bits(f"{tag} {str(dtype)[6:]} store", s.param.detach(),
                             arena_view(ar["M"], lo + s.offset, s.param).to(dtype))
                ck.true(f"{tag} zero_input", bool((s.param.grad == 0).all()), s.name)
        ck.close()


# ============================================================================================ the bounds themselves (CPU)
def _fma32(a, b, c):
    return (a.astype(np.float64) * b + c).astype(np.float32)


def emulate_k7(g, p, s0, s1, h, t, lr, scale, fault=None):
    """K7 in numpy fp32, in the kernel's operation order (fmaf through float64, which rounds twice at most), with
    an optional fault.  Returns (p, s0, s1) as fp32 arrays."""
    f = np.float32
    g = (g * f(scale)).astype(np.float32)
    if h["maximize"] and fault != "maximize ignored":
        g = -g
    p = p.copy()
    if h["kind"] == 1:
        if h["weight_decay"] != 0:
            g = _fma32(f(h["weight_decay"]), p, g)
        b = s0
        if h["momentum"] != 0:
            if t == 0:
                b = (f(1) - f(h["dampening"])) * g if fault == "first-step dampening" else g
            else:
                b = _fma32(f(h["momentum"]), s0, (f(1) - f(h["dampening"])) * g)
            prev = s0 if fault == "nesterov previous buffer" else b
            g = _fma32(f(h["momentum"]), prev, g) if h["nesterov"] else b
        return _fma32(-f(lr), g, p), b, s1
    tt = t if fault == "bias correction at t" else t + 1
    if fault == "fp32 bias correction":
        bc1 = f(1) - np.power(f(h["beta1"]), f(tt))
        bc2 = np.sqrt(f(1) - np.power(f(h["beta2"]), f(tt)))
    else:
        bc1, bc2 = f(1.0 - float(f(h["beta1"])) ** tt), f(math.sqrt(1.0 - float(f(h["beta2"])) ** tt))
    if h["adamw"]:
        lr_d = f(h["lr"]) if fault == "adamw decay ignores lr_scale" else f(lr)
        p = p * (f(1) - lr_d * f(h["weight_decay"]))
    elif h["weight_decay"] != 0:
        g = _fma32(f(h["weight_decay"]), p, g)
    m = _fma32(f(h["beta1"]), s0, (f(1) - f(h["beta1"])) * g)
    v = _fma32(f(h["beta2"]), s1, (f(1) - f(h["beta2"])) * g * g)
    if fault == "eps inside sqrt":
        den = np.sqrt(v + f(h["eps"])) / bc2
    else:
        den = np.sqrt(v) / bc2 + f(h["eps"])
    return _fma32(-(f(lr) / bc1), m / den, p), m, v


def emulate_lamb_dir(g, p, s0, s1, h, t, scale):
    f = np.float32
    g = (g * f(scale)).astype(np.float32)
    bc1, bc2 = f(1.0 - float(f(h["beta1"])) ** (t + 1)), f(math.sqrt(1.0 - float(f(h["beta2"])) ** (t + 1)))
    m = _fma32(f(h["beta1"]), s0, (f(1) - f(h["beta1"])) * g)
    v = _fma32(f(h["beta2"]), s1, (f(1) - f(h["beta2"])) * g * g)
    return _fma32(f(h["weight_decay"]), p, (m / bc1) / (np.sqrt(v) / bc2 + f(h["eps"]))), m, v


def _cpu_case(kind, n=4096, seed=5, t=3, **over):
    """Inputs and fp32 hyperparameters of a CPU check: wide gradients (underflowing squares included), unit
    parameters, and a lr large enough that the update is as large as the parameter."""
    rng = np.random.default_rng(seed)
    g = rng.standard_normal(n)
    k = np.arange(0, n, 3)
    g[k] = np.sign(g[k]) * 10.0 ** rng.uniform(-30, 18, k.size)
    g = g.astype(np.float32)
    p = rng.standard_normal(n).astype(np.float32)
    s0 = (0.1 * rng.standard_normal(n)).astype(np.float32)
    s1 = (0.01 * rng.standard_normal(n) ** 2).astype(np.float32)
    base = dict(kind=1, nesterov=0, adamw=0, maximize=0, lr=0.5, momentum=0.9, dampening=0.3, weight_decay=1e-2,
                beta1=0.9, beta2=0.999, eps=1e-8)
    if kind != "sgd":
        base.update(kind=2 if kind != "lamb" else 4, adamw=int(kind == "adamw"), weight_decay=0.1)
    base.update(over)
    h = {k: (_f32(v) if isinstance(v, float) else v) for k, v in base.items()}
    return g, p, s0, s1, h, t


def _check_cpu(g, p, s0, s1, h, t, lr, scale, outs, dtype=torch.bfloat16):
    """The same checks as the GPU tests on an emulated launch: master, S0 / S1 and the 16-bit store."""
    ck = Checker()
    T = lambda x: torch.from_numpy(np.asarray(x)).double()   # noqa: E731
    ref = k7_ref(T(g), T(p), T(s0), T(s1), h, t, lr, scale)
    tag = "cpu " + {1: "sgd", 2: "adamw" if h["adamw"] else "adam"}[h["kind"]]
    pm, m0, m1, out16 = outs
    ck.bound(f"{tag} master", torch.from_numpy(pm), ref["p"])
    for k, o in (("s0", m0), ("s1", m1)):
        if k in ref:
            ck.bound(f"{tag} {k.upper()}", torch.from_numpy(o), ref[k])
    ck.same_bits(f"{tag} store", out16, torch.from_numpy(pm).to(dtype))
    return ck, ref


def _emulated(kind, fault=None, t=3, lr_scale=1.0, store=None, master_lost=False, **over):
    g, p, s0, s1, h, t = _cpu_case(kind, t=t, **over)
    lr = _f32(np.float32(h["lr"]) * np.float32(lr_scale))
    pm, m0, m1 = emulate_k7(g, p, s0, s1, h, t, lr, 0.125, fault)
    out = torch.from_numpy(pm).to(torch.bfloat16)
    if store == "truncate":
        out = (torch.from_numpy(pm).view(torch.int32) & -65536).view(torch.float32).to(torch.bfloat16)
    if master_lost:
        pm = p.copy()
    return _check_cpu(g, p, s0, s1, h, t, lr, 0.125, (pm, m0, m1, out))


CPU_CONFIGS = {
    "sgd-first": dict(kind="sgd", t=0),
    "sgd-nesterov-max": dict(kind="sgd", nesterov=1, maximize=1),
    "sgd-mom0": dict(kind="sgd", momentum=0.0),
    "adam-l2": dict(kind="adam"),
    "adam-b2-0.99999": dict(kind="adam", beta2=0.99999, t=1),
    "adamw-lrscale-max": dict(kind="adamw", lr_scale=0.3, maximize=1),
}


@pytest.mark.parametrize("name", list(CPU_CONFIGS))
def test_cpu_emulation_within_bounds(name):
    ck, _ = _emulated(**CPU_CONFIGS[name])
    ck.close()


def test_cpu_clip_apply_and_lamb_direction_within_bounds():
    """K9 is K7 on fl(r coef) with scale 1; the LAMB direction of K10."""
    g, p, s0, s1, h, t = _cpu_case("adam")
    r = (g * np.float32(0.125)).astype(np.float32)
    coef = np.float32(0.37)
    gs = (r * coef).astype(np.float32)
    lr = h["lr"]
    pm, m0, m1 = emulate_k7(gs, p, s0, s1, h, t, lr, 1.0)
    ck, _ = _check_cpu(gs, p, s0, s1, h, t, lr, 1.0, (pm, m0, m1, torch.from_numpy(pm).to(torch.bfloat16)))
    g, p, s0, s1, h, t = _cpu_case("lamb")
    d, m0, m1 = emulate_lamb_dir(g, p, s0, s1, h, t, 0.125)
    T = lambda x: torch.from_numpy(np.asarray(x)).double()   # noqa: E731
    ref = lamb_dir_ref(T(g), T(p), T(s0), T(s1), h, t, 0.125)
    ck.bound("cpu lamb direction", torch.from_numpy(d), ref["r"])
    ck.bound("cpu lamb S0", torch.from_numpy(m0), ref["s0"])
    ck.bound("cpu lamb S1", torch.from_numpy(m1), ref["s1"])
    ck.close()


@pytest.mark.parametrize("name", ["sgd-first", "adam-l2", "adamw-lrscale-max"])
def test_cpu_tightest_element_beyond_bound_fails(name):
    """The element closest to its bound, moved to 1.01x the bound (in float64), fails; at 0.99x it passes."""
    cfg = dict(CPU_CONFIGS[name])
    g, p, s0, s1, h, t = _cpu_case(cfg.pop("kind"), t=cfg.pop("t", 3), **{k: v for k, v in cfg.items()
                                                                           if k != "lr_scale"})
    lr = _f32(np.float32(h["lr"]) * np.float32(cfg.get("lr_scale", 1.0)))
    pm = emulate_k7(g, p, s0, s1, h, t, lr, 0.125)[0]
    T = lambda x: torch.from_numpy(np.asarray(x)).double()   # noqa: E731
    ref = k7_ref(T(g), T(p), T(s0), T(s1), h, t, lr, 0.125)["p"]
    ratio = Checker().bound("cpu tightness probe", torch.from_numpy(pm), ref)
    i = int(torch.argmax(ratio))
    assert 0 < float(ratio[i]) <= 1
    for f, ok in ((1.01, False), (0.99, True)):
        moved = T(pm).clone()
        moved[i] = ref.v[i] + f * ref.e[i]
        ck = Checker()
        ck.bound("cpu tightness probe", moved, ref)
        assert (not ck.fails) == ok
    fp64_bounds._WORST.pop("cpu tightness probe", None)


FAULTS = [
    # fault, configuration, group that must catch it
    ("first-step dampening", dict(kind="sgd", t=0), "cpu sgd S0"),
    ("bias correction at t", dict(kind="adam"), "cpu adam master"),
    ("fp32 bias correction", dict(kind="adam", beta2=0.999, t=1, weight_decay=0.0, lr=1.0), "cpu adam master"),
    ("eps inside sqrt", dict(kind="adam"), "cpu adam master"),
    ("adamw decay ignores lr_scale", dict(kind="adamw", lr_scale=0.3), "cpu adamw master"),
    ("nesterov previous buffer", dict(kind="sgd", nesterov=1), "cpu sgd master"),
    ("truncating bf16 store", dict(kind="adam", store="truncate"), "cpu adam store"),
    ("master not written back", dict(kind="sgd", master_lost=True), "cpu sgd master"),
    ("maximize ignored", dict(kind="adamw", maximize=1), "cpu adamw master"),
]


@pytest.mark.parametrize("fault,cfg,group", FAULTS, ids=[f[0] for f in FAULTS])
def test_cpu_fault_is_caught(fault, cfg, group):
    """Each fault, in an fp32 emulation of the kernel, fails the bound of the group it belongs to.  (The fp32
    bias correction is the kernel's code before it formed the corrections in double: at beta2 = 0.999 and step 2
    it is off by about 100 u.)"""
    kw = {"fault": fault} if fault not in ("truncating bf16 store", "master not written back") else {}
    worst = dict(fp64_bounds._WORST)
    ck, _ = _emulated(**cfg, **kw)
    fp64_bounds._WORST.clear()
    fp64_bounds._WORST.update(worst)                  # the faulty run's ratios are not part of the report
    assert any(f.startswith(group + ":") for f in ck.fails), ck.fails or "nothing failed"
