"""LSTM kernel numerics against float64, element by element and one time step at a time: the persistent recurrence
K5 (csrc/lstm_rec_sm90.cu: the forward and backward cluster kernels, ``lstm_xproj_kernel``, ``lstm_wgrad_kernel``,
``lstm_in_mma_kernel`` in its three modes and ``lstm_ih_wgrad_finish_kernel``) and the fused linear head K6
(csrc/lstm_kernels.cu).

The entry points are called directly (``b200dp_lstm_rec_fwd`` / ``_bwd``, ``b200dp_head_fwd`` / ``_bwd``), so the
workspaces autograd hides are checked too: the x-projection ``xp``, the saved post-activation gates, the cell states
``cs`` and the per-step gate gradients ``dG``.  Every output starts as NaN (``dW_hh`` as zero, which its split-K
atomics need), so an element a kernel does not write fails.

An elementwise bound through a whole recurrence would pile up error over the steps.  Instead each step is checked
against float64 computed from the state the kernel itself used at that step: h_{t-1} from its ``seq`` (``h0`` at the
first step of the walk), c_{t-1} from its ``cs`` (or ``c0``), and in the backward pass dh_t from its ``dG`` of the
previous walk step.  The only quantity carried from step to step is the backward cell gradient dc, which the kernel
keeps in registers; its bound is carried with it and shrinks by the forget gate at each step.

Every bound is derived from the roundings the kernel performs (each helper writes its derivation out), not fitted to
observed errors.  u = 2^-24 is the fp32 unit roundoff.  A sum of n fp32 terms in any order is within 2 n u sum|terms|
of the exact sum (the factor 2 covers the tensor cores' internal accumulation).  An fp32 value read as tf32 by wgmma
keeps 10 mantissa bits, truncated or rounded: relative error below 2^-10 either way, so a product of two tf32
operands is within 2 * 2^-10 (+ 2^-20, covered by the accumulation term) of the fp32 product.  Zero-filled K tails
are counted as terms.
"""
import math

import pytest
import torch

import fp64_bounds
from fp64_bounds import U32, assert_within_bound, report_ratios

gpu = pytest.mark.gpu

H = 256                   # hidden size of the kernels
G = 4 * H                 # gate rows (i, f, g, o)
NB = 32                   # batch tile of one cluster
CL = 8                    # CTAs per cluster
SIMT_MAX_F = 32           # inputs up to this width use the fp32 SIMT x-projection / dW_ih / dx kernels

TF32_OP = 2 * 2.0 ** -10  # operand term of a product of two fp32 values read as tf32
ULP = 2.0 ** -23          # one ulp of an fp32 value, relative to its magnitude (at most)
U_DIV = 2 * ULP           # __fdividef: 2 ulp for 2^-126 <= |divisor| <= 2^126 (CUDA C Programming Guide)
FLUSH = 2.0 ** -126       # __expf flushes a subnormal result to 0; __fdividef returns 0 for divisors above 2^126
K_REC_BWD = 128 + CL      # backward dh: a wgmma sum over the CTA's 128 gate rows, then the 8 partials in order


@pytest.fixture(scope="module", autouse=True)
def _report_ratios():
    yield
    report_ratios()


def _cdiv(a, b):
    return -(-a // b)


# ============================================================================================ nonlinearity bounds
def sigmoid_err(lo, hi):
    """Bound on |sigmoidf_fast(x) - sigmoid(x)| for any kernel argument x in [lo, hi] (float64 tensors).

    sigmoidf_fast(x) = __fdividef(1, 1 + __expf(-x)):
    - e = __expf(-x) is within (2 + floor(1.173 |x|)) ulp of exp(-x) (CUDA C Programming Guide), a relative error
      rho_e; 1 + e then moves by rho_e e = rho_e (1 - sigmoid(x)) (1 + e) relative;
    - fl(1 + e): u; __fdividef: 2 ulp (U_DIV);
    - so the result is within sigmoid(x) ((1 - sigmoid(x)) rho_e + u + U_DIV) (1.01 for second-order terms);
    - a subnormal e flushed to 0 moves the result by at most 2^-126, and __fdividef returns 0 for a divisor above
      2^126 (also __expf overflowing to inf), where the exact result is below 2^-126: + 2 * 2^-126 absolute.
    Each factor is taken at its maximum over [lo, hi]."""
    m = torch.maximum(lo.abs(), hi.abs())
    rho_e = (2 + torch.floor(1.173 * m)) * ULP
    return 1.01 * torch.sigmoid(hi) * ((1 - torch.sigmoid(lo)) * rho_e + U32 + U_DIV) + 2 * FLUSH


def tanh_err(lo, hi):
    """Bound on |tanhf_fast(x) - tanh(x)| for x in [lo, hi], in absolute terms: tanhf_fast(x) = 2 s - 1 with
    s = sigmoidf_fast(2 x) (2 x and 2 s are exact).  2 s - 1 cancels near x = 0, so no relative bound holds there:
    the error is 2 sigmoid_err(2 lo, 2 hi), plus u for the subtraction (exact by Sterbenz for s >= 1/4, otherwise
    within u |2 s - 1| <= u)."""
    return 2 * sigmoid_err(2 * lo, 2 * hi) + U32


def _nearest_zero(lo, hi):
    return torch.where(lo > 0, lo, torch.where(hi < 0, hi, torch.zeros_like(lo)))


def gate_bound(pre, E_pre, is_tanh):
    """float64 gate value and bound from a pre-activation known to within E_pre: the nonlinearity's derivative at
    its maximum over [pre - E_pre, pre + E_pre] (both derivatives peak at 0, so at the point of the interval
    nearest to 0) times E_pre, plus the intrinsic error at any argument in that interval."""
    lo, hi = pre - E_pre, pre + E_pre
    z = _nearest_zero(lo, hi)
    if is_tanh:
        return torch.tanh(pre), (1 - torch.tanh(z) ** 2) * E_pre + tanh_err(lo, hi)
    s = torch.sigmoid(z)
    return torch.sigmoid(pre), s * (1 - s) * E_pre + sigmoid_err(lo, hi)


def prod_bound(factors, roundings):
    """float64 product and bound of fl(v_1 ... v_k) when each v_i is known to within E_i (``factors``: (v, E)
    pairs): |prod(v + e) - prod(v)| <= prod(|v| + E) - prod(|v|), and each of the ``roundings`` fp32 roundings
    adds u of the computed magnitude (at most prod(|v| + E)), 1.01 for their compounding."""
    ref, mag, hi = 1.0, 1.0, 1.0
    for v, e in factors:
        ref = ref * v
        mag = mag * v.abs()
        hi = hi * (v.abs() + e)
    return ref, hi - mag + 1.01 * roundings * U32 * hi


# ======================================================================================== per-step references
def prev_state(seq, cs, h0, c0, reverse):
    """The state each step of the walk starts from, [T, B, H] (seq and cs [T, B, H], the kernel's own): h0 / c0 at
    the first step, then the previous step's output (t - 1 going forward, t + 1 for the reverse direction)."""
    if reverse:
        return torch.cat([seq[1:], h0[None]]), torch.cat([cs[1:], c0[None]])
    return torch.cat([h0[None], seq[:-1]]), torch.cat([c0[None], cs[:-1]])


def forward_items(x, h_prev, c_prev, w_ih, w_hh, b_ih, b_hh, xp, gates, cs, seq, tag):
    """(group, out, ref, bound) of every forward output of one direction, each step from the kernel's own state.
    x [T, B, F] as the layer reads it (after inter-layer dropout), h_prev / c_prev [T, B, H] from ``prev_state``;
    xp / gates [T, B, 4H], cs / seq [T, B, H].

    1. xp = x W_ih^T + (b_ih + b_hh).  F <= 32 (lstm_xproj_kernel): fp32 fma chain from fl(b_ih + b_hh), any-order
       bound over n = F + 2 terms.  F > 32 (lstm_in_mma_kernel XPROJ): tf32 operands (TF32_OP), a K of
       32 ceil(F / 32) with the zero tail, then + fl(b_ih + b_hh): n = 32 ceil(F / 32) + 2.
    2. pre = fl(h_{t-1} W_hh^T + xp), the reference computed from x and the weights (not from the kernel's xp, so
       a wrong time or batch index of xp shows): E_pre = (TF32_OP + 2 * 256 u) sum|h||W_hh| + E_xp + u of the sum.
    3. gates: i, f, o = sigmoid(pre), g = tanh(pre), bounded by ``gate_bound``.
    4. c_t = f c_{t-1} + i g from the kernel's saved gates and c_{t-1}: two products and a sum, 4 u (|f c| + |i g|)
       whether or not the compiler fuses them.
    5. h_t = o tanhf_fast(c_t) from the kernel's o and c_t: |o| tanh_err(c_t) + u of the product."""
    X, Hp, Cp = x.double(), h_prev.double(), c_prev.double()
    Wi, Wh = w_ih.double(), w_hh.double()
    F = X.shape[-1]
    Mb = b_ih.double().abs() + b_hh.double().abs()
    Mx = X.abs() @ Wi.abs().t()
    xp_ref = X @ Wi.t() + (b_ih.double() + b_hh.double())
    if F <= SIMT_MAX_F:
        n = F + 2
        E_xp = 2 * n * U32 * (Mx + Mb)
    else:
        n = 32 * _cdiv(F, 32) + 2
        E_xp = (TF32_OP + 2 * n * U32) * Mx + 2 * n * U32 * Mb
    Mh = Hp.abs() @ Wh.abs().t()
    pre = Hp @ Wh.t() + xp_ref
    E_pre = (TF32_OP + 2 * H * U32) * Mh + E_xp + 1.01 * U32 * (Mh + Mx + Mb)
    del Hp, X
    items = [(f"fwd.xp[{tag}]", xp, xp_ref, E_xp)]
    for k, name in enumerate("ifgo"):
        sl = slice(k * H, (k + 1) * H)
        ref, bound = gate_bound(pre[..., sl], E_pre[..., sl], is_tanh=name == "g")
        items.append((f"fwd.gate_{'tanh' if name == 'g' else 'sigmoid'}[{tag}]", gates[..., sl], ref, bound))
    i, f, g, o = gates.double().split(H, -1)
    fc, ig = f * Cp, i * g
    items.append((f"fwd.c[{tag}]", cs, fc + ig, 4 * U32 * (fc.abs() + ig.abs())))
    c = cs.double()
    th, Eth = torch.tanh(c), tanh_err(c, c)
    items.append((f"fwd.h[{tag}]", seq, o * th, o.abs() * Eth + 1.01 * U32 * o.abs() * (th.abs() + Eth)))
    return items


def backward_items(order, w_hh, gates, cs, c_prev, dseq, dhT, dcT, dG, dh0, dc0, tag):
    """(group, out, ref, bound) of the backward recurrence of one direction.  ``order``: the time steps in the
    backward walk's order (the forward walk reversed); gates / dG [T, B, 4H], cs / c_prev / dseq [T, B, H];
    dhT / dcT [B, H] or None.

    1. dh_t = W_hh^T dG_prev + dseq_t, dG_prev the kernel's dG of the previous walk step (dhT + dseq_t at the first
       step): tf32 operands (TF32_OP), and a term goes through the CTA's wgmma sum over its 128 gate rows and the
       fixed-order sum of the 8 cluster partials, 2 (128 + 8) u; then u of the + dseq.
    2. tc = tanhf_fast(c_t): tanh_err (c_t read exactly); A = 1 - tc^2 within (2 |tanh| + E_tc) E_tc + 2.02 u.
    3. dc_t = dc_next + dh o A, dc_next = fl(dc_{t+1} f_{t+1}) (dcT at the first step).  dc_next lives in registers
       only, so its bound is carried: E_dc_t = f_{t+1} E_dc_{t+1} + u |dc_next| + E(dh o A) + u of the sum.  This is
       elementwise and shrinks at each step because 0 < f < 1.
    4. dG: di = dc g i (1 - i), df = dc c_{t-1} f (1 - f), dg = dc i (1 - g^2), do = dh tc o (1 - o) by
       ``prod_bound``; 1 - s is within u |1 - s| (exact for s >= 1/2), 1 - g^2 within 2.02 u (|g| <= 1).
    5. dh0 = W_hh^T dG of the last walk step (as 1.), dc0 = fl(dc f) of the last step (as the carry of 3.)."""
    Wh = w_hh.double()
    i, f, g, o = gates.double().split(H, -1)
    dGk = dG.double()
    R = dGk @ Wh
    Mr = dGk.abs() @ Wh.abs()
    k_rec = TF32_OP + 2 * K_REC_BWD * U32
    first, rest, before = order[0], order[1:], order[:-1]
    rec = torch.zeros_like(R)
    E_rec = torch.zeros_like(R)
    rec[rest] = R[before]
    E_rec[rest] = k_rec * Mr[before]
    if dhT is not None:
        rec[first] = dhT.double()
    ds = dseq.double()
    dh = rec + ds
    E_dh = E_rec + 1.01 * U32 * (rec.abs() + E_rec + ds.abs())
    c = cs.double()
    th, E_tc = torch.tanh(c), tanh_err(c, c)
    A, E_A = 1 - th * th, (2 * th.abs() + E_tc) * E_tc + 2.02 * U32
    P, E_P = prod_bound([(dh, E_dh), (o, 0.0), (A, E_A)], 2)
    dc = torch.empty_like(P)
    E_dc = torch.empty_like(P)
    cn = dcT.double() if dcT is not None else torch.zeros_like(P[0])
    E_cn = torch.zeros_like(cn)
    for s, t in enumerate(order):
        if s:
            fp = f[order[s - 1]]
            cn = fp * dc[order[s - 1]]
            E_cn = fp * E_dc[order[s - 1]] + 1.01 * U32 * (cn.abs() + fp * E_dc[order[s - 1]])
        dc[t] = cn + P[t]
        E_dc[t] = E_cn + E_P[t] + 1.01 * U32 * (cn.abs() + E_cn + P[t].abs() + E_P[t])
    Cp = c_prev.double()
    refs = [prod_bound([(dc, E_dc), (g, 0.0), (i, 0.0), (1 - i, U32 * (1 - i).abs())], 3),
            prod_bound([(dc, E_dc), (Cp, 0.0), (f, 0.0), (1 - f, U32 * (1 - f).abs())], 3),
            prod_bound([(dc, E_dc), (i, 0.0), (1 - g * g, 2.02 * U32)], 2),
            prod_bound([(dh, E_dh), (th, E_tc), (o, 0.0), (1 - o, U32 * (1 - o).abs())], 3)]
    items = [(f"bwd.dG_{name}[{tag}]", dG[..., k * H:(k + 1) * H], ref, bound)
             for k, (name, (ref, bound)) in enumerate(zip("ifgo", refs))]
    last = order[-1]
    items.append((f"bwd.dh0[{tag}]", dh0, R[last], k_rec * Mr[last]))
    fl = f[last]
    dc0_ref = fl * dc[last]
    items.append((f"bwd.dc0[{tag}]", dc0, dc0_ref, fl * E_dc[last] + 1.01 * U32 * (dc0_ref.abs() + fl * E_dc[last])))
    return items


def reduction_items(x_eff, h_prev, dGs, w_ihs, dW_hh, dW_ih, db, dx, keep, scale, tag):
    """(group, out, ref, bound) of the sums over (t, b) and over the gate rows, from the kernel's own dG.
    x_eff [T, B, F] as the layer read it, h_prev [T, B, H] per direction (``prev_state``), dGs / w_ihs / dW_hh /
    dW_ih / db per direction; dx [T, B, F] or None; keep [T, B, F] bool or None (inter-layer dropout of x).

    - dW_hh = sum dG^T h_prev (lstm_wgrad_kernel): fp32 fma chains, split-K partials added with atomics onto 0:
      any order over n = T B + 4 terms.
    - dW_ih, db (= db_ih = db_hh): F <= 32, fp32 SIMT warp sums over n = T B terms, no operand term.  F > 32,
      tf32 wgmma (lstm_in_mma_kernel WGRAD; db against a column of ones, so it too carries the operand term); the
      (t, b) range is split into at most ceil(T B / 128) ranges, each zero-padded by < 32, summed in split order:
      n = T B + 33 ceil(T B / 128).
    - dx = sum_d dG_d W_ih_d: one direction and F <= 32, fp32 SIMT over n = 1024; otherwise tf32 wgmma with K = 1024
      per direction and one add of the two directions: n = 1024 D + 1.  With dropout, dx = scale * sum where x was
      kept (scale = 2 at p = 1/2 is exact) and exactly 0 where it was dropped (checked separately)."""
    X = x_eff.double()
    T, B, F = X.shape
    TB = T * B
    Xf = X.reshape(TB, F)
    items = []
    for d, (dG, Hp) in enumerate(zip(dGs, h_prev)):
        D64 = dG.double().reshape(TB, G)
        Hf = Hp.double().reshape(TB, H)
        items.append((f"bwd.dW_hh[{tag}]", dW_hh[d], D64.t() @ Hf,
                      2 * (TB + 4) * U32 * (D64.abs().t() @ Hf.abs())))
        if F <= SIMT_MAX_F:
            k_ih, k_b, path = 2 * TB * U32, 2 * TB * U32, "simt"
        else:
            n = TB + 33 * _cdiv(TB, 128)
            k_ih = k_b = TF32_OP + 2 * n * U32
            path = "tf32"
        items.append((f"bwd.dW_ih.{path}[{tag}]", dW_ih[d], D64.t() @ Xf, k_ih * (D64.abs().t() @ Xf.abs())))
        items.append((f"bwd.db.{path}[{tag}]", db[d], D64.sum(0), k_b * D64.abs().sum(0)))
    if dx is not None:
        ndir = len(dGs)
        ref = sum(dG.double() @ w.double() for dG, w in zip(dGs, w_ihs))
        mag = sum(dG.double().abs() @ w.double().abs() for dG, w in zip(dGs, w_ihs))
        if ndir == 1 and F <= SIMT_MAX_F:
            k, path = 2 * G * U32, "simt"
        else:
            k, path = TF32_OP + 2 * (G * ndir + 1) * U32, "tf32"
        if keep is not None:
            ref, mag = ref * keep * scale, mag * keep * scale
        items.append((f"bwd.dx.{path}[{tag}]", dx, ref, k * mag))
    return items


def assert_items(items):
    for group, out, ref, bound in items:
        assert_within_bound(out, ref, group=group, terms=[(1.0, bound)])


# ================================================================================================= K5 on a GPU
def _lr():
    from distributed_torch_horovod_gcp_b200.ops import kernels, lstm_rec
    assert kernels.has("lstm_recurrent"), "lstm_rec kernels missing from libb200dp_kernels.so"
    return lstm_rec


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _nan(*shape):
    return torch.full(shape, float("nan"), device="cuda")


def _tb(t):
    """[B, T, C] -> [T, B, C] (the layout of xp, gates, cs and dG)."""
    return t.transpose(0, 1)


def make_inputs(D, B, T, F, regime, seed):
    """Weights with nn.LSTM's init (U(-1/16, 1/16)), x / h0 / c0 / dseq / dhT / dcT standard normal, drawn from a
    seeded CPU generator.  ``saturating``: W_ih x 320 / sqrt(F) and the biases x 16, so pre-activations spread to
    about +-100 whatever F is, and +60 on the i and f biases and on half of the g biases, so those cells grow by
    about 1 per step (to about T); W_hh x 4 only, which keeps the backward recurrence's gain below 1 (a larger
    W_hh makes the exact gradients themselves overflow fp32 within 200 steps).  ``near_zero``: weights, h0 and c0
    x 1e-3, so g and tanh(c) sit where 2 sigmoid(2x) - 1 cancels."""
    g = torch.Generator().manual_seed(seed)
    k = H ** -0.5

    def u(*s):
        return (torch.rand(*s, generator=g) * 2 - 1) * k

    def n(*s):
        return torch.randn(*s, generator=g)

    ws = [[u(G, F), u(G, H), u(G), u(G)] for _ in range(D)]
    x, h0, c0 = n(B, T, F), n(D, B, H), n(D, B, H)
    dseq, dhT, dcT = n(B, T, D * H), n(D, B, H), n(D, B, H)
    if regime == "saturating":
        for w in ws:
            w[0].mul_(320 / math.sqrt(F))
            w[1].mul_(4)
            w[2].mul_(16)
            w[3].mul_(16)
            w[2][:2 * H] += 60
            w[2][2 * H:2 * H + H // 2] += 60
    elif regime == "near_zero":
        for w in ws:
            for t in w:
                t.mul_(1e-3)
        h0.mul_(1e-3)
        c0.mul_(1e-3)
    else:
        assert regime == "default"
    cu = lambda t: t.cuda().contiguous()  # noqa: E731
    return ([[cu(t) for t in w] for w in ws], cu(x), cu(h0), cu(c0), cu(dseq), cu(dhT), cu(dcT))


def run_fwd(x, ws, h0, c0, train=True, p=0.0, in_keep=None, out_seed=None, out_keep=None):
    """One b200dp_lstm_rec_fwd call with every output NaN-filled.  Per direction: dict of xp, gates, cs, hT, cT
    (gates / cs None in inference)."""
    lr = _lr()
    B, T, F = x.shape
    D = len(ws)
    seq = _nan(B, T, D * H)
    outs, ptrs = [], []
    for d, (w_ih, w_hh, b_ih, b_hh) in enumerate(ws):
        o = {"xp": _nan(T, B, G), "gates": _nan(T, B, G) if train else None, "cs": _nan(T, B, H) if train else None,
             "hT": _nan(B, H), "cT": _nan(B, H)}
        outs.append(o)
        # FW_* enum order of csrc/lstm_rec_sm90.cu
        ptrs += [w_ih, w_hh, b_ih, b_hh, h0[d], c0[d], o["xp"], o["gates"], o["cs"], o["hT"], o["cT"]]
    lr._ck(lr._lib.b200dp_lstm_rec_fwd(x.data_ptr(), seq.data_ptr(), lr._ptr_array(ptrs), D, B, T, F, p,
                                       lr._p(in_keep), lr._p(out_seed), lr._p(out_keep), _stream()))
    return seq, outs


def run_bwd(x, seq, ws, h0, c0, fwd, dseq, dhT, dcT, p=0.0, in_keep=None):
    """One b200dp_lstm_rec_bwd call with every output NaN-filled except dW_hh (zero: split-K atomics)."""
    lr = _lr()
    B, T, F = x.shape
    D = len(ws)
    dx = _nan(B, T, F)
    outs, ptrs = [], []
    for d, (w_ih, w_hh, _, _) in enumerate(ws):
        o = {"dG": _nan(T, B, G), "dh0": _nan(B, H), "dc0": _nan(B, H), "dW_ih": _nan(G, F),
             "dW_hh": torch.zeros(G, H, device="cuda"), "db_ih": _nan(G), "db_hh": _nan(G)}
        outs.append(o)
        # BW_* enum order of csrc/lstm_rec_sm90.cu
        ptrs += [w_ih, w_hh, h0[d], c0[d], fwd[d]["gates"], fwd[d]["cs"], dhT[d], dcT[d], o["dG"], o["dh0"],
                 o["dc0"], o["dW_ih"], o["dW_hh"], o["db_ih"], o["db_hh"]]
    lr._ck(lr._lib.b200dp_lstm_rec_bwd(x.data_ptr(), seq.data_ptr(), dseq.data_ptr(), dx.data_ptr(),
                                       lr._ptr_array(ptrs), D, B, T, F, p, lr._p(in_keep), _stream()))
    return dx, outs


def _walk(T, reverse):
    return list(range(T - 1, -1, -1)) if reverse else list(range(T))


def check_layer(x, x_eff, ws, h0, c0, dseq, dhT, dcT, tag, p=0.0, in_keep=None, keep=None):
    """Forward in training and inference mode, then the backward pass of one layer, every output checked.
    x_eff / keep: x as the layer reads it and the dropout mask, [B, T, F]."""
    B, T, F = x.shape
    D = len(ws)
    seq, fwd = run_fwd(x, ws, h0, c0, p=p, in_keep=in_keep)
    seq_i, inf = run_fwd(x, ws, h0, c0, train=False, p=p, in_keep=in_keep)
    torch.cuda.synchronize()
    # the inference forward (nothing saved) takes the same arithmetic path as the training forward
    assert torch.equal(seq_i, seq), "inference seq differs from the training forward"
    hps = []
    for d in range(D):
        assert torch.equal(inf[d]["hT"], fwd[d]["hT"]) and torch.equal(inf[d]["cT"], fwd[d]["cT"]), \
            f"inference h_n / c_n differ from the training forward (direction {d})"
        seq_d = _tb(seq[..., d * H:(d + 1) * H])
        cs = fwd[d]["cs"]
        last = 0 if d else T - 1
        # the final state is the last step of the walk, bit for bit
        assert torch.equal(fwd[d]["hT"], seq_d[last]) and torch.equal(fwd[d]["cT"], cs[last]), \
            f"h_n / c_n are not the last walk step of seq / cs (direction {d})"
        hp, cp = prev_state(seq_d, cs, h0[d], c0[d], reverse=bool(d))
        hps.append(hp)
        assert_items(forward_items(_tb(x_eff), hp, cp, *ws[d], fwd[d]["xp"], fwd[d]["gates"], cs, seq_d, tag))
    dx, bwd = run_bwd(x, seq, ws, h0, c0, fwd, dseq, dhT, dcT, p=p, in_keep=in_keep)
    torch.cuda.synchronize()
    for d in range(D):
        cs = fwd[d]["cs"]
        _, cp = prev_state(_tb(seq[..., d * H:(d + 1) * H]), cs, h0[d], c0[d], reverse=bool(d))
        order = _walk(T, reverse=not d)
        assert_items(backward_items(order, ws[d][1], fwd[d]["gates"], cs, cp, _tb(dseq[..., d * H:(d + 1) * H]),
                                    dhT[d], dcT[d], bwd[d]["dG"], bwd[d]["dh0"], bwd[d]["dc0"], tag))
        assert torch.equal(bwd[d]["db_ih"], bwd[d]["db_hh"]), "db_ih and db_hh differ"
    kp = _tb(keep) if keep is not None else None
    assert_items(reduction_items(_tb(x_eff), hps, [o["dG"] for o in bwd], [w[0] for w in ws],
                                 [o["dW_hh"] for o in bwd], [o["dW_ih"] for o in bwd], [o["db_ih"] for o in bwd],
                                 _tb(dx), kp, 2.0, tag))
    if keep is not None:
        assert bool((dx[~keep] == 0).all()), "dx is not exactly 0 where the input was dropped"


def multi_tile_batch(D):
    """A batch that gives every cluster more than one 32-row tile, with a ragged last tile: cluster_split gives
    each direction (SMs / 8) / D clusters, which walk the tiles with a stride of that count."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    cpd = (sms // CL) // D
    B = NB * (cpd + 1) + 5
    assert _cdiv(B, NB) > cpd and B % NB, (B, cpd)
    return B


# (directions, batch, steps, features, regime): every value of each axis appears at least once.  "multi": a
# batch with more than one tile per cluster (``multi_tile_batch``); 2500: the reference's validation batch.
CASES = [
    (1, 1, 1, 1, "default"),
    (1, 33, 7, 23, "default"),
    (2, 33, 10, 32, "default"),
    (1, "multi", 10, 33, "default"),
    (2, "multi", 7, 100, "default"),
    (1, 2500, 10, 23, "default"),
    (1, 33, 200, 23, "default"),
    (2, 1, 200, 512, "saturating"),
    (1, 33, 10, 23, "saturating"),
    (2, "multi", 10, 23, "saturating"),
    (2, 33, 7, 33, "near_zero"),
    (1, "multi", 200, 100, "near_zero"),
]


@gpu
@pytest.mark.parametrize("D,B,T,F,regime", CASES)
def test_recurrence_per_step(D, B, T, F, regime):
    """K5 forward (training and inference), backward and parameter / input gradients of one layer, each step
    against float64 from the kernel's own state."""
    if B == "multi":
        B = multi_tile_batch(D)
    ws, x, h0, c0, dseq, dhT, dcT = make_inputs(D, B, T, F, regime, seed=1000 * D + 7 * T + F)
    tag = f"{regime},F{'<=' if F <= SIMT_MAX_F else '>'}32"
    check_layer(x, x, ws, h0, c0, dseq, dhT, dcT, tag)


@gpu
@pytest.mark.parametrize("D", [1, 2])
def test_two_layers_with_dropout(D):
    """Two layers with inter-layer dropout p = 1/2 (the DROP instantiations of lstm_in_mma_kernel): layer 0 draws
    the keep mask of its output, layer 1 reads its input through it in the x-projection and dW_ih, and its dx is
    the gradient of layer 0's undropped output, exactly 0 where an element was dropped."""
    B, T, F, p = 33, 7, 23, 0.5
    ws0, x, h0, c0, _, _, _ = make_inputs(D, B, T, F, "default", seed=77 + D)
    ws1, _, h1, c1, dseq, dhT, dcT = make_inputs(D, B, T, D * H, "default", seed=78 + D)
    words = B * T * D * H // 32
    keep_w = torch.empty(words, dtype=torch.int32, device="cuda")
    seed = torch.tensor([0x1234_5678_9ABC, 42], dtype=torch.int64, device="cuda")
    seq0, fwd0 = run_fwd(x, ws0, h0, c0, p=p, out_seed=seed, out_keep=keep_w)
    torch.cuda.synchronize()
    keep = ((keep_w[:, None] >> torch.arange(32, dtype=torch.int32, device="cuda")) & 1).bool().reshape(B, T, D * H)
    frac = float(keep.float().mean())
    assert 0.4 < frac < 0.6, frac
    # layer 0 itself (drawing the mask leaves its arithmetic unchanged)
    for d in range(D):
        seq_d = _tb(seq0[..., d * H:(d + 1) * H])
        hp, cp = prev_state(seq_d, fwd0[d]["cs"], h0[d], c0[d], reverse=bool(d))
        assert_items(forward_items(_tb(x), hp, cp, *ws0[d], fwd0[d]["xp"], fwd0[d]["gates"], fwd0[d]["cs"], seq_d,
                                   "dropout,layer0"))
    x1 = seq0.contiguous()
    check_layer(x1, x1 * keep * 2.0, ws1, h1, c1, dseq, dhT, dcT, "dropout,layer1", p=p, in_keep=keep_w, keep=keep)


# ================================================================================================= K6 on a GPU
def _head_lib():
    from distributed_torch_horovod_gcp_b200.ops import kernels, lstm_fused
    assert kernels.has("lstm_fused"), "fused head kernels missing from libb200dp_kernels.so"
    return lstm_fused


def head_items(x, W, b, a1, a2, pred, dpred, da1, da2, dx, dW, db):
    """(group, out, ref, bound) of the fused head, each stage from the kernel's previous stage.  x [B, K0] is the
    selected time step, W / b the three layers.

    - forward (dense_rows): fp32 fma chains over lanes, a shuffle tree, then + bias: any order over n = K + 1.
      a1 from x, a2 from the kernel's a1, pred from the kernel's a2.
    - backward rows (dense_cols): an fma chain over the layer's outputs: n = N.  da2 from dpred, da1 from the
      kernel's da2, dx from the kernel's da1.
    - weights: dW = sum_b dY^T X (an fma chain over b, n = B), db = sum_b dY (lanes and a shuffle tree, n = B),
      from the kernel's dY and X of each layer."""
    B = x.shape[0]
    ins = [x, a1, a2]
    outs = [a1, a2, pred]
    items = []
    for l in range(3):
        X, Wl, bl = ins[l].double(), W[l].double(), b[l].double()
        n = Wl.shape[1] + 1
        items.append((f"head.fwd_{l + 1}", outs[l], X @ Wl.t() + bl,
                      2 * n * U32 * (X.abs() @ Wl.abs().t() + bl.abs())))
    dys = [dpred, da2, da1]                   # gradient of the output of layer 3, 2, 1
    douts = [da2, da1, dx]
    for l in (2, 1, 0):
        dY, Wl = dys[2 - l].double(), W[l].double()
        items.append((f"head.bwd_rows_{l + 1}", douts[2 - l], dY @ Wl, 2 * Wl.shape[0] * U32 * (dY.abs() @ Wl.abs())))
    for l in range(3):
        dY, X = dys[2 - l].double(), ins[l].double()
        items.append((f"head.dW_{l + 1}", dW[l], dY.t() @ X, 2 * B * U32 * (dY.abs().t() @ X.abs())))
        items.append((f"head.db_{l + 1}", db[l], dY.sum(0), 2 * B * U32 * dY.abs().sum(0)))
    return items


def _head_params(K0, N3, g):
    dims = [(H, K0), (64, H), (N3, 64)]
    W = [((torch.rand(o, i, generator=g) * 2 - 1) * i ** -0.5).cuda() for o, i in dims]
    b = [((torch.rand(o, generator=g) * 2 - 1) * i ** -0.5).cuda() for o, i in dims]
    return W, b


# (batch, input width = 256 x directions, outputs)
HEAD_CASES = [(1, 512, 1), (33, 256, 3), (1024, 256, 1), (1024, 512, 1)]


@gpu
@pytest.mark.parametrize("B,K0,N3", HEAD_CASES)
def test_head_stages(B, K0, N3):
    """K6 forward and backward through the C entry points: every stage against float64 from the kernel's
    previous stage; dx lands at the selected time step of dseq and nowhere else."""
    hf = _head_lib()
    T, t_index = 3, 2
    g = torch.Generator().manual_seed(B + K0 + N3)
    W, b = _head_params(K0, N3, g)
    seq = torch.randn(B, T, K0, generator=g).cuda()
    dpred = torch.randn(B, N3, generator=g).cuda()
    a1, a2, pred = _nan(B, H), _nan(B, 64), _nan(B, N3)
    st = _stream()
    off = t_index * K0 * 4
    hf._ck(hf._lib.b200dp_head_fwd(seq.data_ptr() + off, T * K0, W[0].data_ptr(), b[0].data_ptr(), W[1].data_ptr(),
                                   b[1].data_ptr(), W[2].data_ptr(), b[2].data_ptr(), a1.data_ptr(), a2.data_ptr(),
                                   pred.data_ptr(), B, K0, H, 64, N3, st))
    da1, da2, dseq = _nan(B, H), _nan(B, 64), _nan(B, T, K0)
    dW = [_nan(*w.shape) for w in W]
    db = [_nan(*v.shape) for v in b]
    hf._ck(hf._lib.b200dp_head_bwd(dpred.data_ptr(), seq.data_ptr() + off, T * K0, a1.data_ptr(), a2.data_ptr(),
                                   W[0].data_ptr(), W[1].data_ptr(), W[2].data_ptr(), da1.data_ptr(), da2.data_ptr(),
                                   dseq.data_ptr() + off, T * K0, dW[0].data_ptr(), db[0].data_ptr(),
                                   dW[1].data_ptr(), db[1].data_ptr(), dW[2].data_ptr(), db[2].data_ptr(),
                                   B, K0, H, 64, N3, st))
    torch.cuda.synchronize()
    assert_items(head_items(seq[:, t_index], W, b, a1, a2, pred, dpred, da1, da2, dseq[:, t_index], dW, db))
    others = [t for t in range(T) if t != t_index]
    assert bool(dseq[:, others].isnan().all()), "the head backward wrote dseq outside the selected time step"

    # through the autograd binding: the same bits, and exact zeros at every other step of dseq
    s = seq.clone().requires_grad_()
    out = hf._HeadFn.apply(s, t_index, *[t.clone().requires_grad_() for pair in zip(W, b) for t in pair])
    assert torch.equal(out.reshape(B, N3), pred)
    (ds,) = torch.autograd.grad(out, [s], dpred.reshape(B, 1, N3))
    assert torch.equal(ds[:, t_index], dseq[:, t_index])
    assert bool((ds[:, others] == 0).all()), "dseq is not exactly 0 outside the selected time step"


@gpu
def test_head_rejects_batch_above_1024():
    """The weight-gradient kernel stages one column of dY in 1024 floats of shared memory: B = 1025 is refused
    before any launch."""
    hf = _head_lib()
    g = torch.Generator().manual_seed(3)
    W, b = _head_params(H, 1, g)
    seq = torch.randn(1025, 1, H, device="cuda")
    with pytest.raises(RuntimeError, match="head dims too large"):
        hf._HeadFn.apply(seq, 0, W[0], b[0], W[1], b[1], W[2], b[2])


# ======================================================= the bounds themselves, on a float32 CPU emulation
def _tf32(t):
    """fp32 -> tf32 by truncation (10 explicit mantissa bits)."""
    return (t.float().contiguous().view(torch.int32) & ~0x1FFF).view(torch.float32)


def _emu_sigmoid(x):
    return 1 / (1 + torch.exp(-x))


def _emu_tanh(x):
    return 2 * _emu_sigmoid(2 * x) - 1


def emulate_forward(x, h0, c0, w_ih, w_hh, b_ih, b_hh, fault=None, other_h=None):
    """A float32 emulation of the forward walk (one direction): tf32-truncated recurrent operands, fp32 sums, the
    1 / (1 + exp(-x)) formulas in fp32.  x [T, B, F].  ``fault`` (at step 1 only) feeds the step a wrong state the
    way a broken index would: "batch_row" (h of the neighbouring batch row), "prev_step" (h_{t-2}), "swizzle"
    (two k positions swapped inside a 16-byte group), "other_dir" (``other_h``), "tile" (c of the batch row 32
    away, the next tile)."""
    T = x.shape[0]
    xp = x @ w_ih.t() + (b_ih + b_hh)
    h, c = h0, c0
    hs, cs, gs = [], [], []
    for t in range(T):
        hr, cr = h, c
        if t == 1 and fault == "batch_row":
            hr = h.roll(1, 0)
        elif t == 1 and fault == "prev_step":
            hr = h0
        elif t == 1 and fault == "swizzle":
            hr = h.clone()
            hr[:, [8, 9]] = h[:, [9, 8]]
        elif t == 1 and fault == "other_dir":
            hr = other_h
        elif t == 1 and fault == "tile":
            cr = c.roll(NB, 0)
        pre = _tf32(hr) @ _tf32(w_hh).t() + xp[t]
        i, f, g, o = pre.split(H, -1)
        i, f, g, o = _emu_sigmoid(i), _emu_sigmoid(f), _emu_tanh(g), _emu_sigmoid(o)
        c = f * cr + i * g
        h = o * _emu_tanh(c)
        hs.append(h)
        cs.append(c)
        gs.append(torch.cat([i, f, g, o], -1))
    return xp, torch.stack(gs), torch.stack(cs), torch.stack(hs)


def emulate_backward(w_hh, gates, cs, c_prev, dseq, dhT, dcT):
    """A float32 emulation of the backward walk (forward direction): tf32-truncated operands for W_hh^T dG."""
    T = gates.shape[0]
    dGs = [None] * T
    dh_rec, dc_next = dhT, dcT
    for t in range(T - 1, -1, -1):
        i, f, g, o = gates[t].split(H, -1)
        dh = dh_rec + dseq[t]
        tc = _emu_tanh(cs[t])
        dc = dc_next + dh * o * (1 - tc * tc)
        dG = torch.cat([dc * g * i * (1 - i), dc * c_prev[t] * f * (1 - f), dc * i * (1 - g * g),
                        dh * tc * o * (1 - o)], -1)
        dGs[t] = dG
        dc_next = dc * f
        dh_rec = _tf32(dG) @ _tf32(w_hh)
    return torch.stack(dGs), dh_rec, dc_next


def _emu_inputs(seed, B=64, T=2, F=23):
    g = torch.Generator().manual_seed(seed)
    k = H ** -0.5
    u = lambda *s: (torch.rand(*s, generator=g) * 2 - 1) * k  # noqa: E731
    w = [u(G, F), u(G, H), u(G), u(G)]
    x, h0, c0 = torch.randn(T, B, F, generator=g), torch.randn(B, H, generator=g), torch.randn(B, H, generator=g)
    return w, x, h0, c0, g


def _emu_items(fault=None):
    w, x, h0, c0, g = _emu_inputs(11)
    other = None
    if fault == "other_dir":
        w2, _, h2, c2, _ = _emu_inputs(12)
        other = emulate_forward(x, h2, c2, *w2)[3][0]
    xp, gates, cs, seq = emulate_forward(x, h0, c0, *w, fault=fault, other_h=other)
    hp, cp = prev_state(seq, cs, h0, c0, reverse=False)
    items = forward_items(x, hp, cp, *w, xp, gates, cs, seq, "cpu")
    T, B = x.shape[:2]
    dseq, dhT, dcT = (torch.randn(T, B, H, generator=g), torch.randn(B, H, generator=g),
                      torch.randn(B, H, generator=g))
    dG, dh0, dc0 = emulate_backward(w[1], gates, cs, cp, dseq, dhT, dcT)
    items += backward_items(_walk(T, reverse=True), w[1], gates, cs, cp, dseq, dhT, dcT, dG, dh0, dc0, "cpu")
    return items


class _KeepRatios:
    """Deliberately failing checks must not show up in the module's worst-ratio report."""

    def __enter__(self):
        self.saved = dict(fp64_bounds._WORST)

    def __exit__(self, *exc):
        fp64_bounds._WORST.clear()
        fp64_bounds._WORST.update(self.saved)


def test_emulated_steps_within_bounds():
    """A float32 emulation of a forward step and a backward step (tf32-truncated operands, exact-libm
    nonlinearities) falls inside every bound."""
    with _KeepRatios():
        assert_items(_emu_items())


def test_tightest_element_at_1p01_bound_fails():
    """Each bound is a bound, not a tolerance with slack: the element closest to its bound, moved to 1.01 times
    the bound, fails."""
    with _KeepRatios():
        for group, out, ref, bound in _emu_items():
            err = (out.double() - ref).abs()
            k = int(torch.argmax(err / bound))
            moved = out.double().clone().reshape(-1)
            moved[k] = ref.reshape(-1)[k] + 1.01 * bound.reshape(-1)[k]
            with pytest.raises(AssertionError):
                assert_within_bound(moved.reshape(out.shape), ref, group=group, terms=[(1.0, bound)])


@pytest.mark.parametrize("fault,group", [("batch_row", "fwd.gate"), ("prev_step", "fwd.gate"),
                                         ("swizzle", "fwd.gate"), ("other_dir", "fwd.gate"), ("tile", r"fwd.c\[")])
def test_realistic_fault_is_caught(fault, group):
    """The per-step check finds the faults it exists for in the default regime: one step fed h of the neighbouring
    batch row, of the step before, with two k positions swapped inside a 16-byte swizzle group, of the other
    direction (all in the gate pre-activations), or c of the wrong tile (in the cell update)."""
    items = _emu_items(fault)
    with _KeepRatios(), pytest.raises(AssertionError, match=group):
        assert_items(items)


def test_nonlinearity_bounds_hold_at_fp32_extremes():
    """The sigmoid / tanh bounds at arguments where the intrinsics misbehave: exp(-x) over- or underflowing fp32
    (|x| near 88 and 100), and tanh near 0, where 2 sigmoid(2x) - 1 cancels.  An fp32 emulation with every
    rounding the kernel makes (rounded exp, fp32 1 + e and division, flush to zero) stays inside."""
    x32 = torch.cat([torch.linspace(-110, 110, 20001), torch.logspace(-8, 0, 2001), -torch.logspace(-8, 0, 2001)])
    x = x32.double()
    e = torch.exp(-x32)
    e = torch.where(e < 2.0 ** -126, torch.zeros_like(e), e)
    d = 1 + e
    s = torch.where(d > 2.0 ** 126, torch.zeros_like(d), 1 / d)
    with _KeepRatios():
        assert_within_bound(s, torch.sigmoid(x), group="cpu.sigmoid", terms=[(1.0, sigmoid_err(x, x))])
        th = 2 * _emu_sigmoid(2 * x32) - 1
        assert_within_bound(th, torch.tanh(x), group="cpu.tanh", terms=[(1.0, tanh_err(x, x))])
