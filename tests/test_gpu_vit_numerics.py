"""ViT-B/16 numerics against float64: the flash attention (csrc/attn_sm90.cu) forward, LSE and backward, and
the LayerNorm forward and backward (csrc/elementwise.cu ln_fwd / ln_bwd), element by element, plus the whole
encoder block against an fp64 copy.

Every reference is the operation in float64 on the exact bf16 (or fp32) values the kernel saw.  Every bound
is derived from the roundings the kernel performs (listed in ``attn_fwd_bounds``, ``attn_bwd_bounds`` and
``ln_bounds``), not fitted to observed errors.  The bounds hold for any order of the fp32 atomics (LayerNorm
dgamma / dbeta, attention dQ), so they do not depend on the run being reproducible.

Input regimes are chosen where these kernels go wrong: sequence lengths at every 128-row tile edge, B != H
(swapped batch / head indices), softmax rows peaked across KV blocks (the online rescale ``alpha``), logits
shifted by +-200 natural units (beyond fp32 exp: a running maximum that starts at 0 instead of -inf, or an
overflow, shows), operands in different memory layouts in one call, LayerNorm rows with a large mean (a
one-pass variance fails) and constant rows (variance 0).

Not covered: the cached dQ workspace (``ops.attention._dq_workspace``) is keyed by shape and device but not
by stream; two concurrent backward passes of the same shape on different streams would share it.  No caller
does that today.
"""
import copy
import math

import pytest
import torch
import torch.nn.functional as F

import fp64_bounds
from fp64_bounds import U32, U_BF16, assert_within_bound, report_ratios

gpu = pytest.mark.gpu

LN2 = math.log(2.0)
LOG2E = 1.0 / LN2
# Accuracy of the approximate fp32 instructions, as documented (PTX ISA, CUDA C Programming Guide), with a
# factor of 2 to spare: ex2.approx.ftz.f32 (2 ulp), __fdividef (2 ulp), rsqrtf (2 ulp), log2f (1 ulp).
U_EX2 = 2.0 ** -21
U_DIV = 2.0 ** -21
U_RSQRT = 2.0 ** -21
U_LOG2 = 2.0 ** -22
TILE = 128                # attention query / key tile
BA, HA = 2, 3             # attention batch and heads: B != H, both > 1


@pytest.fixture(scope="module", autouse=True)
def _report_ratios():
    yield
    report_ratios()


def _cdiv(a, b):
    return -(-a // b)


def _t(x):
    return x.transpose(-1, -2)


# ================================================================================================ attention
def attn_ref64(q, k, v):
    """float64 softmax(q k^T / 8) v and the natural-log LSE of the scaled scores, [B, H, S, 64] inputs."""
    q, k, v = q.double(), k.double(), v.double()
    s = q @ _t(k) / 8.0
    lse = torch.logsumexp(s, dim=-1)
    return torch.exp(s - lse[..., None]) @ v, lse


def attn_fwd_bounds(q, k, v, weights_exact=False):
    """float64 o*, lse* and per-element bounds ``terms`` for ``assert_within_bound``.

    The kernel (one query row; x_j = s_j log2(e) / 8 are the exact scaled scores in log2 units):

    1. s~_j: fp32 accumulation of the 64 exact bf16 products, |s~_j - s_j| <= 2*64*u*(|q||k|)_j, times
       c~ = fl(log2(e)/8) (relative error u), minus the running maximum m_b inside one fma (one rounding
       u*|t_j|, |t_j| <= x_max - x_j + 1).  The rescale factors alpha = ex2(m_{b-1} - m_b) telescope, so
       key j's weight is 2^(x_j - m_final) up to an exponent error E_j (log2 units) of those terms plus the
       roundings of the nb - 1 subtractions m_{b-1} - m_b (together <= u*(x_max - x_min + 1)), and up to
       nb + 1 ex2.approx factors (1 + U_EX2).  Relative weight error: eta = max_j 2^E_j (1 + U_EX2)^(nb+1) - 1.
       No weight may flush to zero (ex2.ftz below 2^-126): every case keeps a row's spread below 120 log2 units.
    2. The normalised weights w~_j / sum w~ are within a factor (1 + eta)/(1 - eta) of P*_j, so
       |sum_j w~_j v_j / sum w~ - o*| <= 2 eta/(1 - eta) * (P*|V|).  With V constant along the sequence this
       term is 0 (``weights_exact``).
    3. P~ is rounded to bf16 before P V (relative U_BF16 per term) while l sums the unrounded fp32 values.
    4. O: fp32 accumulation of S products plus nb rescales, 2*(S + nb)*u relative to sum |P~||V|;
       l: 2*(S + nb + 2)*u (two quad-shuffle adds); 1/l by __fdividef (U_DIV); o*inv (u).
    5. the bf16 store: U_BF16 * |o| <= U_BF16 * (|o*| + |o - o*|).

    Together: |o - o*| <= c1 * (P*|V|) + U_BF16 * |o*|, c1 per row.

    LSE = (m_final + log2f(l)) * fl(ln 2): log2(l) + m_final = log2(sum_j 2^x_j) + log2(1 + eta') +
    log2(1 + eps_l) with |eta'| <= eta, log2f within U_LOG2 * (log2(S) + 1) (|log2 l| <= log2 S + 1), then
    three roundings relative to |lse|: |lse - lse*| <= c1' + 4u * |lse*|."""
    q, k, v = q.detach(), k.detach(), v.detach()
    q64, k64, v64 = q.double(), k.double(), v.double()
    S = q.shape[2]
    nb = _cdiv(S, TILE)
    o, lse = attn_ref64(q, k, v)
    s = q64 @ _t(k64) / 8.0
    p = torch.exp(s - lse[..., None])
    x = s * LOG2E
    xmax = x.amax(-1, keepdim=True)
    xmin = x.amin(-1, keepdim=True)
    assert float((xmax - xmin).max()) < 120.0, "a softmax weight could flush to zero: the bound does not apply"
    ds = 2 * 64 * U32 * (q64.abs() @ _t(k64.abs()))
    E = (LOG2E / 8.0) * ds * (1 + U32) + U32 * x.abs() + U32 * (xmax - x + 1) + U32 * (xmax - xmin + 1)
    eta = torch.expm1(LN2 * E.amax(-1, keepdim=True) + (nb + 1) * math.log1p(U_EX2))
    assert float(eta.max()) < 0.1
    w = torch.zeros_like(eta) if weights_exact else 2 * eta / (1 - eta)
    eps_acc = 2 * (S + nb) * U32
    eps_l = 2 * (S + nb + 2) * U32
    phi = (1 + eps_l / (1 - eps_l)) * (1 + U_DIV) * (1 + U32) - 1
    c_z = w + (U_BF16 + eps_acc * (1 + U_BF16)) * (1 + w) + phi * (1 + w) * (1 + U_BF16) * (1 + eps_acc)
    o_terms = [((1 + U_BF16) * c_z, p @ v64.abs()), (U_BF16, o.abs())]
    c_lse = LN2 * (-torch.log2(1 - eta) - math.log2(1 - eps_l) + U_LOG2 * (math.log2(S) + 1)) * (1 + 4 * U32)
    c_lse = c_lse.squeeze(-1)
    lse_terms = [(c_lse, torch.ones_like(lse)), (4 * U32, lse.abs())]
    lse_bound = c_lse + 4 * U32 * lse.abs()
    return o, lse, o_terms, lse_terms, lse_bound


def attn_bwd_bounds(q, k, v, do, o_k):
    """float64 gradients (autograd through ``attn_ref64``) and per-element bounds for dq, dk, dv.

    ``o_k`` is the output the kernel stored (bf16): the backward computes delta from it.  The kernel:

    1. P~ = ex2(fma(s~, c~, -lse2)), lse2 = fl(LSE * fl(log2 e)) from the forward's LSE (bound of
       ``attn_fwd_bounds``, plus two roundings).  Exponent error E = c*|s~ - s|(1 + u) + u|x| + u(|x - lse2| + 1)
       + |lse2 - lse2*|, so |P~ - P*| <= pi P*, pi = (2^E - 1)(1 + U_EX2) + U_EX2 (pi = 1 where P* may flush).
    2. dV = sum_i bf16(P~) dO_i: fp32 over S terms, then the bf16 store.
    3. dP~ = dO V^T, 64-term fp32 (2*64*u*|dO||V|); delta~ = rowsum(dO o_k) in fp32 from the kernel's bf16
       O: |delta~ - delta*| <= |rowsum(dO (o_k - o*))| + 2*64*u*rowsum|dO||o_k|; g = dP - delta (one rounding).
    4. dS~ = bf16(P~ g~ / 8) (one rounding, /8 exact, then bf16): G >= |dS~ - dS*|.
    5. dQ = dS~ K: fp32 over 128 keys per block, nb blocks summed by fp32 atomics in any order
       (2*(S + nb)*u), bf16 cast; dK = dS~^T Q: fp32 over S rows, bf16 store."""
    q64, k64, v64 = [t.detach().double().requires_grad_(True) for t in (q, k, v)]
    do64 = do.double()
    o, lse = attn_ref64(q64, k64, v64)
    o.backward(do64)
    dq, dk, dv = q64.grad, k64.grad, v64.grad
    q64, k64, v64, o, lse = q64.detach(), k64.detach(), v64.detach(), o.detach(), lse.detach()
    S = q.shape[2]
    nb = _cdiv(S, TILE)
    _, _, _, _, lse_bound = attn_fwd_bounds(q, k, v)
    s = q64 @ _t(k64) / 8.0
    P = torch.exp(s - lse[..., None])
    x = s * LOG2E
    lse2 = (lse * LOG2E)[..., None]
    bl2 = (LOG2E * lse_bound * (1 + U32))[..., None] + 2 * U32 * lse2.abs()
    ds = 2 * 64 * U32 * (q64.abs() @ _t(k64.abs()))
    E = (LOG2E / 8.0) * ds * (1 + U32) + U32 * x.abs() + U32 * ((x - lse2).abs() + 1) + bl2
    pi = torch.expm1(LN2 * E) * (1 + U_EX2) + U_EX2
    pi = torch.where(x - lse2 - E < -125.0, pi.clamp_min(1.0), pi)
    Pe = P * pi
    Phi = P + Pe
    ado = do64.abs()
    dv_b = (1 + U_BF16) * (_t(Pe) @ ado + (U_BF16 + 2 * S * U32 * (1 + U_BF16)) * (_t(Phi) @ ado)) \
        + U_BF16 * dv.abs()
    dP = do64 @ _t(v64)
    dp_err = 2 * 64 * U32 * (ado @ _t(v64.abs()))
    ok64 = o_k.double()
    delta = (do64 * o).sum(-1)
    d_err = (do64 * (ok64 - o)).sum(-1).abs() + 2 * 64 * U32 * (ado * ok64.abs()).sum(-1)
    g = dP - delta[..., None]
    g_err = dp_err + d_err[..., None]
    g_err = g_err + 1.01 * U32 * (g.abs() + g_err)
    dS = P * g / 8.0
    G = (1 + U_BF16) / 8.0 * (Pe * g.abs() + Phi * g_err + U32 * Phi * (g.abs() + g_err)) + U_BF16 * dS.abs()
    Hm = dS.abs() + G
    dq_b = (1 + U_BF16) * (G @ k64.abs() + 2 * (S + nb) * U32 * (Hm @ k64.abs())) + U_BF16 * dq.abs()
    dk_b = (1 + U_BF16) * (_t(G) @ q64.abs() + 2 * S * U32 * (_t(Hm) @ q64.abs())) + U_BF16 * dk.abs()
    return (dq, dq_b), (dk, dk_b), (dv, dv_b)


def attn_inputs(S, regime, seed, B=BA, H=HA):
    """q, k, v [B, H, S, 64] bf16, generated on the CPU (the same values on every machine).

    plain:    q, k, v ~ N(0, 1): logits with standard deviation 1.
    peaked:   logits over the first KV block span about +-25 (standard deviation 7); for S > 128 every key of
              a later block carries a per-(b, h) bonus that puts every row's maximum in a later block, 2 or more
              units above the first block's maximum, so alpha rescales a non-trivial O and l.
    shift+ / shift-: dimension 0 of q is 16 and of every key +-100, which shifts every logit by +-200.
    """
    g = torch.Generator().manual_seed(seed)
    shape = (B, H, S, 64)
    q, k, v = (torch.randn(shape, generator=g) for _ in range(3))
    if regime == "peaked":
        q[..., :32] *= 7.0 * 8.0 / math.sqrt(32.0)
        q[..., 32:] = 0.0
        k[..., 32:] = 0.0
        q[..., 32] = 8.0                               # logit bonus of a key = its dimension 32
        if S > TILE:
            k[:, :, TILE:, :32] *= 0.3
            qb, kb = q.bfloat16().double(), k.bfloat16().double()
            first = (qb @ _t(kb[:, :, :TILE]) / 8.0).amax(-1)                  # [B, H, S]
            later = (qb @ _t(kb[:, :, TILE:]) / 8.0).amax(-1)
            bonus = (first.amax(-1) - later.amin(-1) + 2.0).ceil()             # [B, H], exact in bf16
            k[:, :, TILE:, 32] = bonus[..., None]
    elif regime in ("shift+", "shift-"):
        q[..., 0] = 16.0
        k[..., 0] = 100.0 if regime == "shift+" else -100.0
    else:
        assert regime == "plain"
    return [t.bfloat16() for t in (q, k, v)]


def attn_layout(t, kind, slot=0):
    """A [B, H, S, 64] tensor with t's values in memory layout ``kind``; the rest of its buffer is NaN.

    bhsd:   contiguous [B, H, S, 64];
    bshd:   a [B, S, H, 64] view of a [B*S, H*64] matrix (the model's q / k / v / o);
    packed: slot ``slot`` of a packed [B, S, 3, H, 64] buffer;
    sbhd:   a view of a contiguous [S, B, H, 64] buffer."""
    B, H, S, D = t.shape
    kw = dict(dtype=t.dtype, device=t.device)
    if kind == "bhsd":
        return t.clone(memory_format=torch.contiguous_format)
    if kind == "bshd":
        view = torch.full((B * S, H * D), float("nan"), **kw).view(B, S, H, D).transpose(1, 2)
    elif kind == "packed":
        view = torch.full((B, S, 3, H, D), float("nan"), **kw)[:, :, slot].transpose(1, 2)
    else:
        assert kind == "sbhd"
        view = torch.full((S, B, H, D), float("nan"), **kw).permute(1, 2, 0, 3)
    view.copy_(t)
    return view


QKV_LAYOUTS = [("bhsd", "bshd", "packed"), ("bshd", "packed", "bhsd"), ("packed", "bhsd", "bshd")]


def _qkv_in_layouts(q, k, v, i):
    lq, lk, lv = QKV_LAYOUTS[i % len(QKV_LAYOUTS)]
    return attn_layout(q, lq, 0), attn_layout(k, lk, 1), attn_layout(v, lv, 2)


def _attn():
    from distributed_torch_horovod_gcp_b200.ops import attention, kernels
    assert kernels.has("attention_fused"), "attention kernels missing from libb200dp_kernels.so"
    return attention


def _attn_fwd(q, k, v):
    """``b200dp_attn_fwd`` called directly, with an LSE buffer; o in [B, S, H, 64] memory order."""
    A = _attn()
    B, H, S, D = q.shape
    o = torch.full((B, S, H, D), float("nan"), dtype=torch.bfloat16, device="cuda").permute(0, 2, 1, 3)
    lse = torch.full((B, H, S), float("nan"), dtype=torch.float32, device="cuda")
    A._ck(A._lib.b200dp_attn_fwd(q.data_ptr(), k.data_ptr(), v.data_ptr(), o.data_ptr(), lse.data_ptr(),
                                 B, H, S, D, A._strides(q), A._strides(k), A._strides(v), A._strides(o), 0.125,
                                 torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    return o, lse


ATTN_S = [1, 2, 63, 64, 65, 127, 128, 129, 197, 255, 256, 257, 1024]
REGIMES = ["plain", "peaked", "shift+", "shift-"]


def _check_fwd(q, k, v, o, lse, group, weights_exact=False):
    o64, lse64, o_terms, lse_terms, _ = attn_fwd_bounds(q, k, v, weights_exact)
    assert_within_bound(o, o64, group=f"attn fwd o ({group})", terms=o_terms)
    assert_within_bound(lse, lse64, group=f"attn fwd lse ({group})", terms=lse_terms)


@gpu
@pytest.mark.parametrize("regime", REGIMES)
@pytest.mark.parametrize("S", ATTN_S)
def test_attention_fwd_vs_fp64(S, regime):
    q, k, v = [t.cuda() for t in attn_inputs(S, regime, seed=S)]
    if regime == "peaked" and S > TILE:
        s = q.double() @ _t(k.double())
        assert bool((s.argmax(-1) >= TILE).all()), "every row's maximum must lie past the first KV block"
    qi, ki, vi = _qkv_in_layouts(q, k, v, S)
    o, lse = _attn_fwd(qi, ki, vi)
    _check_fwd(q, k, v, o, lse, regime)


@gpu
@pytest.mark.parametrize("S", [1, 129, 257, 1024])
def test_attention_fwd_constant_v(S):
    """V constant along the sequence (a different row per (b, h)): o equals it up to the P and output
    roundings, whatever the softmax weights are."""
    q, k, v = [t.cuda() for t in attn_inputs(S, "peaked", seed=S + 1)]
    v = v[:, :, :1].expand_as(v).contiguous()
    o, lse = _attn_fwd(*_qkv_in_layouts(q, k, v, S))
    _check_fwd(q, k, v, o, lse, "constant v", weights_exact=True)


@gpu
@pytest.mark.parametrize("S", [1, 65, 300, 1024])
def test_attention_fwd_dominant_key(S):
    """One key per (b, h), at a different position in each, 60 logit units above all others: the other
    weights are below e^-50, the dominant one rounds to exactly 1 in bf16, so o is that key's v row bit
    for bit."""
    g = torch.Generator().manual_seed(S + 2)
    q = torch.randn(BA, HA, S, 64, generator=g)
    k = torch.randn(BA, HA, S, 64, generator=g)
    v = torch.randn(BA, HA, S, 64, generator=g)
    q[..., 0] = 32.0
    k[..., 0] = 0.0
    pos = torch.tensor([[(37 * (b * HA + h) + 11) % S for h in range(HA)] for b in range(BA)])
    for b in range(BA):
        for h in range(HA):
            k[b, h, pos[b, h], 0] = 16.0
    q, k, v = [t.bfloat16().cuda() for t in (q, k, v)]
    s = q.double() @ _t(k.double()) / 8.0
    top2 = s.topk(min(2, S), dim=-1).values
    if S > 1:
        assert float((top2[..., 0] - top2[..., 1]).min()) > 55.0
    o, lse = _attn_fwd(*_qkv_in_layouts(q, k, v, S + 1))
    _check_fwd(q, k, v, o, lse, "dominant key")
    want = torch.stack([torch.stack([v[b, h, pos[b, h]] for h in range(HA)]) for b in range(BA)])
    assert torch.equal(o, want[:, :, None].expand_as(o)), "o is not the dominant key's v row"


def _workspace_zero():
    A = _attn()
    return all(float(w.abs().max()) == 0.0 for w in A._ws.values())


def _check_bwd(q, k, v, do, o, grads, group):
    (dq, dq_b), (dk, dk_b), (dv, dv_b) = attn_bwd_bounds(q, k, v, do, o)
    for name, got, ref, b in (("dq", grads[0], dq, dq_b), ("dk", grads[1], dk, dk_b), ("dv", grads[2], dv, dv_b)):
        if got is not None:
            assert_within_bound(got, ref, group=f"attn bwd {name} ({group})", terms=[(1.0, b)])


def _attn_fwd_bwd(q, k, v, i, need=(True, True, True)):
    """The autograd path (``attention_fused``) with q, k, v in three different layouts and dO in a fourth."""
    A = _attn()
    leaves = [attn_layout(t.detach(), lay, slot).requires_grad_(r)
              for t, lay, slot, r in zip((q, k, v), QKV_LAYOUTS[i % 3], (0, 1, 2), need)]
    o = A.attention_fused(*leaves)
    gen = torch.Generator().manual_seed(1000 + i)
    do = torch.randn(q.shape, generator=gen).bfloat16().cuda()
    o.backward(attn_layout(do, "sbhd"))
    torch.cuda.synchronize()
    return o.detach(), do, [t.grad for t in leaves]


@gpu
@pytest.mark.parametrize("regime", REGIMES)
@pytest.mark.parametrize("S", ATTN_S)
def test_attention_bwd_vs_fp64(S, regime):
    q, k, v = [t.cuda() for t in attn_inputs(S, regime, seed=S)]
    o, do, grads = _attn_fwd_bwd(q, k, v, S)
    _check_bwd(q, k, v, do, o, grads, regime)
    assert _workspace_zero(), "the dQ workspace was left non-zero"


@gpu
@pytest.mark.parametrize("need", [(True, False, False), (False, True, True), (False, False, True)])
def test_attention_bwd_partial_requires_grad(need):
    q, k, v = [t.cuda() for t in attn_inputs(197, "peaked", seed=5)]
    o, do, grads = _attn_fwd_bwd(q, k, v, 2, need)
    assert [gr is not None for gr in grads] == list(need)
    _check_bwd(q, k, v, do, o, grads, "partial")


@gpu
def test_attention_bwd_interleaved_shapes_workspace():
    """Backward passes of two shapes, interleaved: each shape's cached fp32 dQ workspace must be zero when
    its next backward starts accumulating into it."""
    cases = [(197, 2, 3), (256, 3, 2)]
    data = [[t.cuda() for t in attn_inputs(S, "plain", seed=40 + S, B=B, H=H)] for S, B, H in cases]
    for rep in range(2):
        for i, (q, k, v) in enumerate(data):
            o, do, grads = _attn_fwd_bwd(q, k, v, rep + i)
            _check_bwd(q, k, v, do, o, grads, "interleaved")
            assert _workspace_zero()


# ================================================================================================ LayerNorm
def ln_ref64(x, w, b, eps):
    x, w, b = x.double(), w.double(), b.double()
    mu = x.mean(-1, keepdim=True)
    var = ((x - mu) ** 2).mean(-1, keepdim=True)
    return (x - mu) / torch.sqrt(var + eps) * w + b


def ln_bounds(x, w, b, dy, eps):
    """float64 y*, dx*, dgamma*, dbeta* and their per-element bounds, for [R, C] inputs.

    Forward, one warp per row, lane-sequential sums then a 5-level shuffle tree (depth n_r = 8*C/256 + 5):
    mean m~ = fl(fl(sum x) * fl(1/C)): |m~ - mu| <= Em = 1.01*n_r*u*mean|x| + 2.1u|mu|;
    var~ = fl(sum fl(x - m~)^2 * fl(1/C)) + eps = (var + (m~ - mu)^2)(1 +- (n_r + 5)*1.01u) + eps, one more
    rounding; rsqrtf (U_RSQRT): rs = r*(1 + rho);
    y = bf16(fma(fl(fl(x - m~) rs), g, b)): |y - y*| <= (1+U_BF16)(1+u)[(f-1)|g xhat*| + f r* Em |g|]
    + (U_BF16 + u(1+U_BF16))|y*|, f = (1 + rho)(1 + u)^2.  The Em term is what a constant row needs.

    Backward with the saved m~, rs: xh~ = fl(fl(x - m~) rs) within Dxh = (f-1)|xhat*| + f r* Em;
    s1 = mean(dy g), s2 = mean(dy g xh~), same reduction depth; dx = bf16(rs (dy g - s1 - xh~ s2)) with
    three roundings inside.  dgamma / dbeta: R-term fp32 sums in any order (2*R*u*sum|.|), dgamma from xh~
    (sum |dy| Dxh), and a bf16 store for bf16 parameters."""
    x64, g, bb, dy64 = x.double(), w.double(), b.double(), dy.double()
    R, C = x64.shape
    n_r = 8 * (C // 256) + 5
    mu = x64.mean(-1, keepdim=True)
    d = x64 - mu
    var = (d * d).mean(-1, keepdim=True)
    r = 1.0 / torch.sqrt(var + eps)
    xh = d * r
    y = xh * g + bb
    Em = 1.01 * n_r * U32 * x64.abs().mean(-1, keepdim=True) + 2.1 * U32 * mu.abs()
    nu = (1.01 * Em ** 2 + 1.01 * (n_r + 5) * U32 * (var + Em ** 2) + 1.01 * U32 * (var + eps)) / (var + eps)
    assert float(nu.max()) < 0.1
    rho = (1 + nu / (2 * (1 - nu))) * (1 + U_RSQRT) - 1
    f = (1 + rho) * (1 + U32) ** 2
    y_terms = [((1 + U_BF16) * (1 + U32) * (f - 1), (g * xh).abs()),
               ((1 + U_BF16) * (1 + U32) * f * r * Em, g.abs().expand_as(y)),
               (U_BF16 + U32 * (1 + U_BF16), y.abs())]
    dyh = dy64 * g
    s1 = dyh.mean(-1, keepdim=True)
    s2 = (dyh * xh).mean(-1, keepdim=True)
    t = dyh - s1 - xh * s2
    dx = r * t
    Dxh = xh.abs() * (f - 1) + Em * r * f
    Ds1 = 1.02 * (n_r + 4) * U32 * dyh.abs().mean(-1, keepdim=True)
    Ds2 = (1 + U32) * (dyh.abs() * Dxh).mean(-1, keepdim=True) \
        + 1.02 * (n_r + 4) * U32 * (dyh.abs() * (xh.abs() + Dxh)).mean(-1, keepdim=True)
    Dt = Ds1 + xh.abs() * Ds2 + Dxh * (s2.abs() + Ds2) \
        + 3.03 * U32 * (dyh.abs() + s1.abs() + Ds1 + (xh.abs() + Dxh) * (s2.abs() + Ds2))
    fr = (1 + rho) * (1 + U32)
    dx_b = (1 + U_BF16) * (r * fr * Dt + (fr - 1) * dx.abs()) + U_BF16 * dx.abs()
    ady = dy64.abs()
    db = dy64.sum(0)
    db_b = 2 * R * U32 * ady.sum(0)
    dg = (dy64 * xh).sum(0)
    dg_b = (ady * Dxh).sum(0) + 2 * R * U32 * (ady * (xh.abs() + Dxh)).sum(0)
    if w.dtype == torch.bfloat16:
        db_b = (1 + U_BF16) * db_b + U_BF16 * db.abs()
        dg_b = (1 + U_BF16) * dg_b + U_BF16 * dg.abs()
    return y, y_terms, (dx, dx_b), (dg, dg_b), (db, db_b)


def ln_inputs(R, C, regime, pdtype, seed):
    """x [R, C] bf16, gamma / beta in ``pdtype`` (fp32 values are not bf16-representable), dy bf16.

    plain:     x = 2 N(0, 1) + 0.5;
    bigmean:   x = 64 + 0.25 N(0, 1) (E[x^2] - mean^2 cancels 16 bits);
    constant:  every row one value (variance 0, rstd = 1/sqrt(eps))."""
    g = torch.Generator().manual_seed(seed)
    if regime == "plain":
        x = 2 * torch.randn(R, C, generator=g) + 0.5
    elif regime == "bigmean":
        x = 64 + 0.25 * torch.randn(R, C, generator=g)
    else:
        assert regime == "constant"
        x = (4 * torch.randn(R, 1, generator=g)).expand(R, C).contiguous()
    w = torch.rand(C, generator=g) + 0.5
    b = 0.1 * torch.randn(C, generator=g)
    dy = torch.randn(R, C, generator=g)
    return x.bfloat16(), w.to(pdtype), b.to(pdtype), dy.bfloat16()


LN_EPS = 1e-6
LN_C = [256, 512, 768, 1024]
# 9000 rows exceed both grid caps (reduce_grid() * 4 * 16 = 8448 forward, * 2 * 16 = 4224 backward on 132 SMs)
LN_R = [1, 15, 16, 17, 9000]


@gpu
@pytest.mark.parametrize("layout", ["contiguous", "cls"])
@pytest.mark.parametrize("regime", ["plain", "bigmean", "constant"])
@pytest.mark.parametrize("pdtype", [torch.bfloat16, torch.float32], ids=["bf16", "fp32"])
@pytest.mark.parametrize("R", LN_R)
@pytest.mark.parametrize("C", LN_C)
def test_layer_norm_vs_fp64(C, R, pdtype, regime, layout):
    """LayerNorm forward and backward on the kernel path.  ``cls``: x is ``t[:, 0]`` of a [R, 3, C] tensor,
    as the final ViT LayerNorm takes the class token."""
    from distributed_torch_horovod_gcp_b200.ops import counters, ln
    x, w, b, dy = ln_inputs(R, C, regime, pdtype, seed=C + R)
    x, w, b, dy = [t.cuda() for t in (x, w, b, dy)]
    if layout == "cls":
        base = torch.full((R, 3, C), float("nan"), dtype=torch.bfloat16, device="cuda")
        base[:, 0] = x
    else:
        base = x.clone()
    base.requires_grad_(True)
    xin = base[:, 0] if layout == "cls" else base
    wk, bk = w.clone().requires_grad_(True), b.clone().requires_grad_(True)
    assert ln.supported(xin, wk, bk)
    c0 = counters.snapshot()
    y = ln.layer_norm(xin, wk, bk, LN_EPS)
    y.backward(dy)
    torch.cuda.synchronize()
    assert counters.snapshot().get("ln_bwd", 0) > c0.get("ln_bwd", 0)
    y64, y_terms, (dx, dx_b), (dg, dg_b), (db, db_b) = ln_bounds(x, w, b, dy, LN_EPS)
    tag = f"{regime}, {'bf16' if pdtype == torch.bfloat16 else 'fp32'} params"
    assert_within_bound(y, y64, group=f"ln fwd y ({tag})", terms=y_terms)
    gx = base.grad[:, 0] if layout == "cls" else base.grad
    assert_within_bound(gx, dx, group=f"ln bwd dx ({tag})", terms=[(1.0, dx_b)])
    if layout == "cls":
        assert float(base.grad[:, 1:].abs().max()) == 0.0
    assert wk.grad.dtype == pdtype and bk.grad.dtype == pdtype
    assert_within_bound(wk.grad, dg, group=f"ln bwd dgamma ({tag})", terms=[(1.0, dg_b)])
    assert_within_bound(bk.grad, db, group=f"ln bwd dbeta ({tag})", terms=[(1.0, db_b)])


@gpu
@pytest.mark.parametrize("wdtype,bdtype", [(torch.bfloat16, torch.float32), (torch.float32, torch.bfloat16)],
                         ids=["bf16-weight-fp32-bias", "fp32-weight-bf16-bias"])
def test_layer_norm_mixed_param_dtypes(wdtype, bdtype):
    """The kernels read gamma and beta in one dtype: a bias in another dtype must not reach them (it would
    be read as the weight's dtype); ``F2.layer_norm`` must still compute what ``F.layer_norm`` does.  The
    bias sits at the start of a buffer twice its size, so a kernel that reads it as fp32 stays inside it."""
    from distributed_torch_horovod_gcp_b200.ops import functional as F2
    x, w, _, _ = ln_inputs(64, 768, "plain", wdtype, seed=9)
    _, _, b, _ = ln_inputs(64, 768, "plain", bdtype, seed=10)
    x, w = x.cuda(), w.cuda()
    b = torch.cat([b, torch.zeros_like(b)]).cuda()[:768]
    y = F2.layer_norm(x, w, b, LN_EPS)
    ref = F.layer_norm(x, (768,), w.bfloat16(), b.bfloat16(), LN_EPS)
    assert y.dtype == torch.bfloat16
    assert float((y.float() - ref.float()).abs().max()) <= 2 * U_BF16 * float(ref.float().abs().max())


# ================================================================================================ encoder block
def _rel(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm().clamp_min(1e-30))


@gpu
def test_vit_encoder_block_vs_fp64():
    """One ViT-B encoder block (768 wide, 12 heads, MLP 3072, B = 2, S = 197) in bf16: output, input gradient
    and all 12 parameter gradients against a float64 copy of the same bf16 parameters.  The kernel path (split
    QKV GEMM, attention in the model layout both ways, residual linear, LayerNorm, fused MLP) must be at most
    twice as far from it as the same block on PyTorch's bf16 ops, or within one bf16 rounding (2^-8)."""
    from distributed_torch_horovod_gcp_b200.models.vit import EncoderBlock
    from distributed_torch_horovod_gcp_b200.ops import counters, functional as F2
    _attn()
    torch.manual_seed(21)
    blk = EncoderBlock(768, 12, 3072)
    with torch.no_grad():
        for ln_mod in (blk.ln_1, blk.ln_2):
            ln_mod.weight.copy_(1 + 0.2 * torch.randn(768))
            ln_mod.bias.copy_(0.2 * torch.randn(768))
    blk = blk.cuda().to(torch.bfloat16)
    x = torch.randn(2, 197, 768, device="cuda").to(torch.bfloat16)
    gy = torch.randn(2, 197, 768, device="cuda").to(torch.bfloat16)

    def run(m, dtype, reference):
        m = copy.deepcopy(m).to(dtype)
        xin = x.to(dtype, copy=True).requires_grad_(True)
        F2._FORCE_REFERENCE = reference
        try:
            y = m(xin)
            y.backward(gy.to(dtype))
        finally:
            F2._FORCE_REFERENCE = False
        torch.cuda.synchronize()
        return [("out", y.detach()), ("dx", xin.grad)] + [(n, p.grad) for n, p in m.named_parameters()]

    ref = run(blk, torch.float64, True)
    lib = run(blk, torch.bfloat16, True)
    c0 = counters.snapshot()
    ker = run(blk, torch.bfloat16, False)
    c1 = counters.snapshot()
    for op in ("attn_fwd", "attn_bwd", "ln_fwd", "ln_bwd"):
        assert c1.get(op, 0) > c0.get(op, 0), f"{op} did not run"
    assert len(ref) == 14
    bad = []
    for (name, r), (_, lb), (_, kr) in zip(ref, lib, ker):
        assert kr.dtype == torch.bfloat16
        e_lib, e_ker = _rel(lb, r), _rel(kr, r)
        print(f"\n[vit block] {name:12s} rel err vs fp64: library {e_lib:.3e} kernels {e_ker:.3e}", end="")
        assert e_lib < 4 * U_BF16, f"{name}: the library path itself is off ({e_lib:.3e}): the comparison is vacuous"
        if not e_ker <= max(2.0 * e_lib, U_BF16):
            bad.append((name, e_lib, e_ker))
    print()
    assert not bad, f"kernel path more than 2x the library's error: {bad}"


# ================================================================================================ CPU self-checks
def test_attention_reference_matches_sdpa_fp64():
    q, k, v = [t.double().requires_grad_(True) for t in attn_inputs(130, "peaked", seed=3)]
    o, lse = attn_ref64(q, k, v)
    q2, k2, v2 = [t.detach().clone().requires_grad_(True) for t in (q, k, v)]
    o2 = F.scaled_dot_product_attention(q2, k2, v2)
    assert torch.allclose(o, o2, rtol=1e-12, atol=1e-12)
    assert torch.allclose(lse, torch.logsumexp(q.detach() @ _t(k.detach()) / 8.0, -1), rtol=1e-13, atol=1e-13)
    gen = torch.Generator().manual_seed(4)
    do = torch.randn(o.shape, generator=gen, dtype=torch.float64)
    o.backward(do)
    o2.backward(do)
    for a, b2 in ((q, q2), (k, k2), (v, v2)):
        assert torch.allclose(a.grad, b2.grad, rtol=1e-10, atol=1e-12)


def test_layer_norm_reference_matches_torch_fp64():
    x, w, b, _ = ln_inputs(33, 768, "bigmean", torch.float32, seed=5)
    y = ln_ref64(x, w, b, LN_EPS)
    y2 = F.layer_norm(x.double(), (768,), w.double(), b.double(), LN_EPS)
    assert torch.allclose(y, y2, rtol=1e-12, atol=1e-12)
    y3, *_ = ln_bounds(x, w, b, torch.zeros_like(x), LN_EPS)
    assert torch.allclose(y3, y2, rtol=1e-12, atol=1e-12)


def _must_fail(fn):
    with pytest.raises(AssertionError):
        fn()
    fp64_bounds._WORST.pop("perturbed", None)


def test_attention_bounds_accept_fp32_and_reject_perturbed():
    """An fp32 CPU evaluation of the same attention lies inside the kernel bounds; the same result moved by
    3 bf16 ulps (of one element, the one whose bound is tightest) does not."""
    S = 200
    g = torch.Generator().manual_seed(6)
    q, k, v = attn_inputs(S, "plain", seed=6)
    q = (q.float() * 3).bfloat16()                                  # moderately peaked rows
    qf, kf, vf = [t.float().requires_grad_(True) for t in (q, k, v)]
    s = qf @ _t(kf) / 8.0
    o32 = torch.softmax(s, -1) @ vf
    lse32 = torch.logsumexp(s.detach(), -1)
    do = torch.randn(o32.shape, generator=g).bfloat16()
    o32.backward(do.float())
    o64, lse64, o_terms, lse_terms, _ = attn_fwd_bounds(q, k, v)
    assert_within_bound(o32.detach(), o64, group="cpu self-check", terms=o_terms)
    assert_within_bound(lse32, lse64, group="cpu self-check", terms=lse_terms)
    o_k = o32.detach().bfloat16()
    (dq, dq_b), (dk, dk_b), (dv, dv_b) = attn_bwd_bounds(q, k, v, do, o_k)
    for got, ref, b in ((qf.grad, dq, dq_b), (kf.grad, dk, dk_b), (vf.grad, dv, dv_b)):
        assert_within_bound(got, ref, group="cpu self-check", terms=[(1.0, b)])
    bound = sum(c * m for c, m in o_terms)
    for got, ref, b in ((o32.detach(), o64, bound), (qf.grad, dq, dq_b), (kf.grad, dk, dk_b), (vf.grad, dv, dv_b)):
        i = int(torch.argmin(b / ref.abs().clamp_min(1e-30)))
        bad = got.clone().reshape(-1)
        bad[i] += 3 * 2.0 ** -7 * float(ref.reshape(-1)[i].abs())
        _must_fail(lambda: assert_within_bound(bad.view_as(got), ref, group="perturbed", terms=[(1.0, b)]))


def test_layer_norm_bounds_accept_fp32_and_reject_perturbed():
    for regime in ("plain", "bigmean", "constant"):
        x, w, b, dy = ln_inputs(17, 768, regime, torch.bfloat16, seed=7)
        xf, wf, bf = [t.float().requires_grad_(True) for t in (x, w, b)]
        y32 = F.layer_norm(xf, (768,), wf, bf, LN_EPS)
        y32.backward(dy.float())
        y64, y_terms, (dx, dx_b), (dg, dg_b), (db, db_b) = ln_bounds(x, w, b, dy, LN_EPS)
        assert_within_bound(y32.detach(), y64, group="cpu self-check", terms=y_terms)
        for got, ref, bnd in ((xf.grad, dx, dx_b), (wf.grad, dg, dg_b), (bf.grad, db, db_b)):
            assert_within_bound(got, ref, group="cpu self-check", terms=[(1.0, bnd)])
        y_b = sum(c * m for c, m in y_terms)
        for got, ref, bnd in ((y32.detach(), y64, y_b), (xf.grad, dx, dx_b)):
            i = int(torch.argmin(bnd / ref.abs().clamp_min(1e-30)))
            bad = got.clone().reshape(-1)
            bad[i] += 3 * 2.0 ** -7 * float(ref.reshape(-1)[i].abs())
            _must_fail(lambda: assert_within_bound(bad.view_as(got), ref, group="perturbed", terms=[(1.0, bnd)]))
