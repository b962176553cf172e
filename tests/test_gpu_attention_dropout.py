"""Dropout inside the flash-attention kernels (csrc/attn_sm90.cu, ``DROPOUT = true``), the fused dropout +
residual add (csrc/elementwise.cu ``dropout_add_kernel``) and the GPT / ViT models that use them.

1. The mask: a numpy Philox4x32-10 written from the mapping in the kernel's header reproduces, bit for bit,
   the keep mask the kernel applied.  With Q = K = 0 every unmasked probability is non-zero, and with V rows
   j0 .. j0 + 63 one-hot (all other rows zero), output column c of query row i is non-zero exactly when key
   j0 + c is kept for row i; shifting j0 covers any S.
2. O, LSE, dQ, dK and dV against float64 attention under that numpy mask, element by element, with bounds
   derived as in ``test_gpu_causal_attention`` plus the roundings of the dropout scale.
3. Seeds: ``torch.manual_seed`` reproduces the bits, other seeds and CUDA-graph replays draw new ones, and the
   kept fraction over 1.6e7 elements is within 6 sigma of the keep probability.
4. ``dropout_add`` forward and backward bit for bit against the formula under the numpy mask.
5. p = 0 runs the kernels without dropout; the models train eagerly and CUDA-graphed with no SDPA call, and in
   eval mode, or with dropout 0, compute what the models without dropout compute, bit for bit.
"""
import math
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TESTS = os.path.dirname(os.path.abspath(__file__))
for _p in (ROOT, TESTS):
    if _p not in sys.path:
        sys.path.insert(0, _p)

from fp64_bounds import U32, U_BF16, assert_within_bound, report_ratios  # noqa: E402
from test_gpu_vit_numerics import LN2, LOG2E, U_DIV, U_EX2, U_LOG2, attn_inputs, attn_layout  # noqa: E402

gpu = pytest.mark.gpu
TILE = 128
M32 = np.uint64(0xFFFFFFFF)


@pytest.fixture(scope="module", autouse=True)
def _report_ratios():
    yield
    report_ratios()


def _t(x):
    return x.transpose(-1, -2)


def _attn():
    from distributed_torch_horovod_gcp_b200.ops import attention, kernels
    assert kernels.has("attention_fused"), "attention kernels missing from libb200dp_kernels.so"
    return attention


# ================================================================================================ numpy spec
def philox(c0, c1, c2, c3, k0, k1):
    """Philox4x32-10 on uint64 arrays holding 32-bit values; returns the four output words."""
    c0, c1, c2, c3 = [np.asarray(c, dtype=np.uint64) & M32 for c in (c0, c1, c2, c3)]
    c0, c1, c2, c3 = np.broadcast_arrays(c0, c1, c2, c3)
    k0, k1 = np.uint64(k0) & M32, np.uint64(k1) & M32
    for _ in range(10):
        p0 = np.uint64(0xD2511F53) * c0
        p1 = np.uint64(0xCD9E8D57) * c2
        c0, c1, c2, c3 = (p1 >> np.uint64(32)) ^ c1 ^ k0, p1 & M32, (p0 >> np.uint64(32)) ^ c3 ^ k1, p0 & M32
        k0 = (k0 + np.uint64(0x9E3779B9)) & M32
        k1 = (k1 + np.uint64(0xBB67AE85)) & M32
    return c0, c1, c2, c3


def thr16(p):
    return min(65536, max(0, int(math.floor((1.0 - p) * 65536.0 + 0.5))))


def scale16(p):
    t = thr16(p)
    return 65536.0 / t if t else 0.0


def _seed_words(seed):
    s = [int(x) & (2 ** 64 - 1) for x in seed.cpu().tolist()]
    return s[0] & 0xFFFFFFFF, s[0] >> 32, s[1]


def attn_mask(seed, B, H, S, p):
    """[B, H, S, S] bool keep mask of the attention dropout, from the mapping in attn_sm90.cu's header."""
    k0, k1, off = _seed_words(seed)
    t = thr16(p)
    r = np.arange(S, dtype=np.uint64)[:, None]
    c = np.arange(S, dtype=np.uint64)[None, :]
    ctr0 = np.uint64(4) * (c // np.uint64(16)) + (c % np.uint64(8)) // np.uint64(2)
    ctr1 = np.uint64(8) * (r // np.uint64(16)) + r % np.uint64(8)
    word = (np.uint64(2) * ((r // np.uint64(8)) % np.uint64(2)) + (c // np.uint64(8)) % np.uint64(2)).astype(np.int64)
    hi = (c % np.uint64(2)) == 1
    out = np.empty((B, H, S, S), dtype=bool)
    for b in range(B):
        for h in range(H):
            u = np.stack(philox(ctr0, ctr1, b * H + h, off & 0xFFFFFFFF, k0, k1))      # [4, S, S]
            w = np.take_along_axis(u, np.broadcast_to(word, (S, S))[None], 0)[0]
            bits = np.where(hi, w >> np.uint64(16), w & np.uint64(0xFFFF))
            out[b, h] = bits < np.uint64(t)
    return torch.from_numpy(out)


def flat_mask(seed, n, p):
    """[n] bool keep mask of dropout_add, from the mapping in elementwise.cu."""
    k0, k1, off = _seed_words(seed)
    e = np.arange(n, dtype=np.uint64)
    g = e // np.uint64(8)
    u = np.stack(philox(g & M32, g >> np.uint64(32), off & 0xFFFFFFFF, off >> 32, k0, k1))
    w = np.take_along_axis(u, ((e % np.uint64(8)) // np.uint64(2)).astype(np.int64)[None], 0)[0]
    bits = np.where(e % np.uint64(2) == 1, w >> np.uint64(16), w & np.uint64(0xFFFF))
    return torch.from_numpy(bits < np.uint64(thr16(p)))


def test_philox_known_answer():
    # Random123's published known-answer vector for philox4x32_10 (counter and key all ones-bits)
    out = philox(0xFFFFFFFF, 0xFFFFFFFF, 0xFFFFFFFF, 0xFFFFFFFF, 0xFFFFFFFF, 0xFFFFFFFF)
    assert [int(x) for x in out] == [0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD]


# ================================================================================================ kernel calls
def _seed(*vals):
    return torch.tensor(list(vals), dtype=torch.int64, device="cuda")


def _fwd(q, k, v, causal, seed, p):
    """``b200dp_attn_fwd_dropout`` called directly; o in [B, S, H, 64] order, LSE saved."""
    A = _attn()
    B, H, S, D = q.shape
    o = torch.full((B, S, H, D), float("nan"), dtype=torch.bfloat16, device="cuda").permute(0, 2, 1, 3)
    lse = torch.full((B, H, S), float("nan"), dtype=torch.float32, device="cuda")
    A._ck(A._lib.b200dp_attn_fwd_dropout(q.data_ptr(), k.data_ptr(), v.data_ptr(), o.data_ptr(), lse.data_ptr(),
                                         B, H, S, D, A._strides(q), A._strides(k), A._strides(v), A._strides(o),
                                         0.125, int(causal), seed.data_ptr(), p,
                                         torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    return o, lse


def recover_mask(B, H, S, causal, seed, p, layout="bhsd"):
    """The keep mask the forward kernel applied, read back through one-hot V rows (64 keys per call).
    Entries the kernel cannot see (masked by causality) are returned as False."""
    q = attn_layout(torch.zeros(B, H, S, 64, dtype=torch.bfloat16, device="cuda"), layout, 0)
    k = attn_layout(torch.zeros(B, H, S, 64, dtype=torch.bfloat16, device="cuda"), layout, 1)
    out = torch.zeros(B, H, S, S, dtype=torch.bool)
    for j0 in range(0, S, 64):
        n = min(64, S - j0)
        v0 = torch.zeros(B, H, S, 64, dtype=torch.bfloat16, device="cuda")
        v0[:, :, j0 + torch.arange(n), torch.arange(n)] = 1.0
        o, _ = _fwd(q, k, attn_layout(v0, layout, 2), causal, seed, p)
        assert bool(torch.isfinite(o.float()).all())
        out[:, :, :, j0:j0 + n] = (o[..., :n] != 0).cpu()
    return out


def _visible(S, causal):
    return torch.ones(S, S, dtype=torch.bool).tril() if causal else torch.ones(S, S, dtype=torch.bool)


# ================================================================================================ 1. the mask
@gpu
@pytest.mark.parametrize("B,H,S,layout", [(1, 1, 1, "bhsd"), (2, 3, 63, "bshd"), (1, 2, 129, "packed"),
                                          (2, 2, 256, "bhsd"), (1, 1, 300, "sbhd"), (1, 2, 1024, "bshd")])
@pytest.mark.parametrize("causal", [False, True])
def test_mask_matches_spec(B, H, S, layout, causal):
    seed = _seed(0x0123456789ABCDEF, 0x1122334455667788 + S)
    got = recover_mask(B, H, S, causal, seed, 0.5, layout)
    want = attn_mask(seed, B, H, S, 0.5) & _visible(S, causal)
    assert torch.equal(got, want), f"{int((got != want).sum())} of {got.numel()} keep bits differ from the spec"


# ================================================================================================ 2. numerics
def _future(S, device):
    return torch.ones(S, S, dtype=torch.bool, device=device).triu(1)


def ref64(q, k, v, keep, causal, scale):
    """float64 dropout attention (keep and scale fixed) and the natural-log LSE of the un-dropped scores."""
    q, k, v = q.double(), k.double(), v.double()
    s = q @ _t(k) / 8.0
    if causal:
        s = s.masked_fill(_future(q.shape[2], q.device), float("-inf"))
    lse = torch.logsumexp(s, dim=-1)
    return (torch.exp(s - lse[..., None]) * (keep.double() * scale)) @ v, lse


def fwd_bounds(q, k, v, keep, causal, scale):
    """``causal_fwd_bounds`` of test_gpu_causal_attention (the same terms; the row sum l and LSE are the
    un-dropped ones) with P* |V| taken over the kept keys and scaled by 1/q, and the normalisation factor phi
    widened by two fp32 roundings: 2^16 / t rounded to fp32, and its product with 1 / l."""
    q, k, v = q.detach(), k.detach(), v.detach()
    q64, k64, v64 = q.double(), k.double(), v.double()
    S = q.shape[2]
    nb = -(-S // TILE)
    fut = _future(S, q.device) if causal else torch.zeros(S, S, dtype=torch.bool, device=q.device)
    Z = keep.double() * scale
    o, lse = ref64(q, k, v, keep, causal, scale)
    s = q64 @ _t(k64) / 8.0
    p = torch.exp(s - lse[..., None]).masked_fill(fut, 0.0)
    x = s * LOG2E
    xmax = x.masked_fill(fut, float("-inf")).amax(-1, keepdim=True)
    xmin = x.masked_fill(fut, float("inf")).amin(-1, keepdim=True)
    assert float((xmax - xmin).max()) < 120.0, "a softmax weight could flush to zero: the bound does not apply"
    ds = 2 * 64 * U32 * (q64.abs() @ _t(k64.abs()))
    E = (LOG2E / 8.0) * ds * (1 + U32) + U32 * x.abs() + U32 * (xmax - x + 1) + U32 * (xmax - xmin + 1)
    E = E.masked_fill(fut, 0.0)
    eta = torch.expm1(LN2 * E.amax(-1, keepdim=True) + (nb + 1) * math.log1p(U_EX2))
    assert float(eta.max()) < 0.1
    w = 2 * eta / (1 - eta)
    eps_acc = 2 * (S + nb) * U32
    eps_l = 2 * (S + nb + 2) * U32
    phi = (1 + eps_l / (1 - eps_l)) * (1 + U_DIV) * (1 + U32) ** 3 - 1
    c_z = w + (U_BF16 + eps_acc * (1 + U_BF16)) * (1 + w) + phi * (1 + w) * (1 + U_BF16) * (1 + eps_acc)
    o_terms = [((1 + U_BF16) * c_z, (p * Z) @ v64.abs()), (U_BF16, o.abs())]
    c_lse = LN2 * (-torch.log2(1 - eta) - math.log2(1 - eps_l) + U_LOG2 * (math.log2(S) + 1)) * (1 + 4 * U32)
    c_lse = c_lse.squeeze(-1)
    lse_terms = [(c_lse, torch.ones_like(lse)), (4 * U32, lse.abs())]
    return o, lse, o_terms, lse_terms, c_lse + 4 * U32 * lse.abs()


def bwd_bounds(q, k, v, do, o_k, keep, causal, scale):
    """``causal_bwd_bounds`` of test_gpu_causal_attention under the mask:
    - dV = fl(fl(2^16/t) * sum over kept P dO): the un-scaled sum has the bound of the un-dropped kernel over the
      kept products, and the scale adds two fp32 roundings;
    - g = Z dP - D: dP's error is scaled by 1/q (with the two roundings of fl(dP fl(2^16/t))), and D is the
      row sum of dO o O over the kernel's dropped O; dS = P g / 8 and dQ, dK follow as without dropout."""
    q64, k64, v64 = [t.detach().double().requires_grad_(True) for t in (q, k, v)]
    do64 = do.double()
    o, lse = ref64(q64, k64, v64, keep, causal, scale)
    o.backward(do64)
    dq, dk, dv = q64.grad, k64.grad, v64.grad
    q64, k64, v64, o, lse = q64.detach(), k64.detach(), v64.detach(), o.detach(), lse.detach()
    S = q.shape[2]
    nb = -(-S // TILE)
    vis = ~_future(S, q.device) if causal else torch.ones(S, S, dtype=torch.bool, device=q.device)
    M = keep.double()
    Z = M * scale
    *_, lse_bound = fwd_bounds(q, k, v, keep, causal, scale)
    s = q64 @ _t(k64) / 8.0
    P = torch.exp(s - lse[..., None]) * vis
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
    r2 = (1 + U32) ** 2
    e_a = _t(M * Pe) @ ado + (U_BF16 + 2 * S * U32 * (1 + U_BF16)) * (_t(M * Phi) @ ado)
    dv_b = (1 + U_BF16) * (scale * r2 * e_a + (r2 - 1) * dv.abs()) + U_BF16 * dv.abs()
    dP = do64 @ _t(v64)
    dp_err = 2 * 64 * U32 * (ado @ _t(v64.abs()))
    ok64 = o_k.double()
    delta = (do64 * o).sum(-1)
    d_err = (do64 * (ok64 - o)).sum(-1).abs() + 2 * 64 * U32 * (ado * ok64.abs()).sum(-1)
    g = Z * dP - delta[..., None]
    g_err = Z * dp_err * r2 + (r2 - 1) * (Z * dP).abs() + d_err[..., None]
    g_err = g_err + 1.01 * U32 * (g.abs() + g_err)
    dS = P * g / 8.0
    G = (1 + U_BF16) / 8.0 * (Pe * g.abs() + Phi * g_err + U32 * Phi * (g.abs() + g_err)) + U_BF16 * dS.abs()
    Hm = dS.abs() + G
    dq_b = (1 + U_BF16) * (G @ k64.abs() + 2 * (S + nb) * U32 * (Hm @ k64.abs())) + U_BF16 * dq.abs()
    dk_b = (1 + U_BF16) * (_t(G) @ q64.abs() + 2 * S * U32 * (_t(Hm) @ q64.abs())) + U_BF16 * dk.abs()
    return (dq, dq_b), (dk, dk_b), (dv, dv_b)


def _fused(q, k, v, do, causal, p, layout, seed_val):
    """``attention_fused`` forward + backward after ``torch.manual_seed(seed_val)``; returns O, the grads and
    the seed the forward drew (the first device draw after the manual seed)."""
    A = _attn()
    leaves = [attn_layout(t.detach(), layout, slot).requires_grad_(True) for slot, t in enumerate((q, k, v))]
    torch.manual_seed(seed_val)
    o = A.attention_fused(*leaves, causal=causal, dropout_p=p)
    torch.manual_seed(seed_val)
    seed = torch.randint(0, 2 ** 62, (2,), dtype=torch.int64, device="cuda")
    o.backward(attn_layout(do, layout))
    torch.cuda.synchronize()
    return o.detach(), [t.grad for t in leaves], seed


NUM_S = [1, 63, 127, 128, 129, 1024, 2048]


@gpu
@pytest.mark.parametrize("p", [0.1, 0.5])
@pytest.mark.parametrize("causal", [False, True])
@pytest.mark.parametrize("S", NUM_S)
def test_fwd_bwd_vs_fp64(S, causal, p):
    B, H = (1, 2) if S >= 1024 else (2, 3)
    q, k, v = [t.cuda() for t in attn_inputs(S, "plain", seed=S + 1, B=B, H=H)]
    do = torch.randn(q.shape, generator=torch.Generator().manual_seed(S)).bfloat16().cuda()
    layout = "bshd" if S % 2 else "bhsd"
    o, grads, seed = _fused(q, k, v, do, causal, p, layout, 1000 + S)
    keep = attn_mask(seed, B, H, S, p).cuda()
    scale = scale16(p)
    # O through the direct entry point too, to check the LSE it saves
    o_d, lse = _fwd(*[attn_layout(t, layout) for t in (q, k, v)], causal, seed, p)
    assert torch.equal(o_d, o)
    o64, lse64, o_terms, lse_terms, _ = fwd_bounds(q, k, v, keep, causal, scale)
    tag = f"{'causal' if causal else 'full'} p={p}"
    assert_within_bound(o, o64, group=f"dropout fwd o ({tag})", terms=o_terms)
    assert_within_bound(lse, lse64, group=f"dropout fwd lse ({tag})", terms=lse_terms)
    for name, got, (ref, b) in zip(("dq", "dk", "dv"), grads, bwd_bounds(q, k, v, do, o, keep, causal, scale)):
        assert_within_bound(got, ref, group=f"dropout bwd {name} ({tag})", terms=[(1.0, b)])


@gpu
@pytest.mark.parametrize("causal", [False, True])
@pytest.mark.parametrize("S", NUM_S)
def test_p1_gives_exact_zeros(S, causal):
    q, k, v = [t.cuda() for t in attn_inputs(S, "plain", seed=S + 5, B=1, H=2)]
    do = torch.randn(q.shape, generator=torch.Generator().manual_seed(S)).bfloat16().cuda()
    o, grads, _ = _fused(q, k, v, do, causal, 1.0, "bhsd", 7)
    for t in (o, *grads):
        assert not bool(torch.isnan(t).any())
        assert float(t.abs().max()) == 0.0


# ================================================================================================ 3. seeds, graphs
@gpu
def test_manual_seed_reproduces_and_seeds_differ():
    A = _attn()
    q, k, v = [t.cuda() for t in attn_inputs(256, "plain", seed=3)]
    outs = []
    for s in (11, 11, 12):
        torch.manual_seed(s)
        outs.append(A.attention_fused(q, k, v, dropout_p=0.3))
    assert torch.equal(outs[0], outs[1])
    assert not torch.equal(outs[0], outs[2])


@gpu
def test_graph_replays_draw_new_masks():
    A = _attn()
    q, k, v = [t.cuda() for t in attn_inputs(256, "plain", seed=4)]
    g = torch.cuda.CUDAGraph()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        A.attention_fused(q, k, v, causal=True, dropout_p=0.2)
    torch.cuda.current_stream().wait_stream(side)
    with torch.cuda.graph(g):
        out = A.attention_fused(q, k, v, causal=True, dropout_p=0.2)
    seen = []
    for _ in range(3):
        g.replay()
        torch.cuda.synchronize()
        seen.append(out.clone())
    assert not torch.equal(seen[0], seen[1]) and not torch.equal(seen[1], seen[2])


@gpu
def test_kept_fraction_within_6_sigma():
    p = 0.1
    B, H, S = 2, 8, 1024                                   # 1.68e7 elements
    got = recover_mask(B, H, S, False, _seed(987654321, 42), p)
    n = got.numel()
    q = thr16(p) / 65536.0
    sigma = math.sqrt(n * q * (1 - q))
    assert abs(int(got.sum()) - n * q) < 6 * sigma


# ================================================================================================ 4. dropout_add
@gpu
@pytest.mark.parametrize("with_residual", [False, True])
@pytest.mark.parametrize("n,p", [(8, 0.5), (4096 * 768, 0.1), (1000 * 8, 0.9), (64, 1.0)])
def test_dropout_add_bits(n, p, with_residual):
    from distributed_torch_horovod_gcp_b200.ops import dropout as D
    assert D.supported(torch.zeros(8, dtype=torch.bfloat16, device="cuda"), None)
    g = torch.Generator().manual_seed(n)
    y = torch.randn(n, generator=g).bfloat16().cuda().requires_grad_(True)
    r = torch.randn(n, generator=g).bfloat16().cuda().requires_grad_(True) if with_residual else None
    dout = torch.randn(n, generator=g).bfloat16().cuda()
    torch.manual_seed(n)
    out = D.dropout_add(y, r, p)
    torch.manual_seed(n)
    seed = torch.randint(0, 2 ** 62, (2,), dtype=torch.int64, device="cuda")
    out.backward(dout)
    torch.cuda.synchronize()
    keep = flat_mask(seed, n, p).cuda()
    sc = torch.tensor(scale16(p), dtype=torch.float32, device="cuda")    # 2^16 / t rounded to fp32, as the kernel
    d = torch.where(keep, y.detach().float() * sc, torch.zeros((), device="cuda"))
    want = (r.detach().float() + d if with_residual else d).bfloat16()
    assert torch.equal(out.view(torch.int16), want.view(torch.int16))
    dy = torch.where(keep, dout.float() * sc, torch.zeros((), device="cuda")).bfloat16()
    assert torch.equal(y.grad.view(torch.int16), dy.view(torch.int16))
    if with_residual:
        assert torch.equal(r.grad, dout)


# ================================================================================================ 5. p = 0, models
@gpu
def test_p0_runs_the_kernels_without_dropout():
    from distributed_torch_horovod_gcp_b200.ops import counters
    A = _attn()
    q, k, v = [t.cuda().requires_grad_(True) for t in attn_inputs(200, "plain", seed=6)]
    c0 = counters.snapshot()
    o = A.attention_fused(q, k, v, causal=True, dropout_p=0.0)
    o.sum().backward()
    torch.cuda.synchronize()
    c1 = counters.snapshot()
    d = {key: c1.get(key, 0) - c0.get(key, 0) for key in set(c0) | set(c1)}
    assert d.get("attn_fwd") == 1 and d.get("attn_bwd") == 3
    assert not d.get("attn_fwd_dropout") and not d.get("attn_bwd_dropout") and not d.get("dropout_add")


def _no_sdpa(monkeypatch):
    import torch.nn.functional as F

    def _raise(*a, **kw):
        raise AssertionError("F.scaled_dot_product_attention was called on the kernel path")
    monkeypatch.setattr(F, "scaled_dot_product_attention", _raise)


def _gpt_batch():
    g = torch.Generator(device="cuda").manual_seed(2)
    return (torch.randint(0, 512, (4, 128), generator=g, device="cuda"),
            torch.randint(0, 512, (4 * 128,), generator=g, device="cuda"))


def _vit_batch():
    g = torch.Generator(device="cuda").manual_seed(3)
    return (torch.randn(4, 3, 64, 64, generator=g, device="cuda").bfloat16(),
            torch.randint(0, 10, (4,), generator=g, device="cuda"))


def _models():
    from distributed_torch_horovod_gcp_b200.models import gpt_tiny, vit_tiny
    return {
        "gpt": (lambda p: gpt_tiny(dropout=p), _gpt_batch),
        # image 64 / patch 8: 65 tokens; 2 heads of 64 so attention runs on the kernel
        "vit": (lambda p: vit_tiny(image_size=64, dim=128, heads=2, mlp_dim=256, dropout=p, attention_dropout=p),
                _vit_batch),
    }


@gpu
@pytest.mark.parametrize("name", ["gpt", "vit"])
def test_model_trains_eager_and_graphed(name, hvd_single, monkeypatch):
    import torch.nn.functional as F
    from distributed_torch_horovod_gcp_b200.ops import counters
    from distributed_torch_horovod_gcp_b200.utils.graph import GraphedStep
    monkeypatch.setenv("B200DP_FUSED_SINGLE", "1")
    hvd = hvd_single
    _attn()
    make, batch = _models()[name]
    torch.manual_seed(0)
    m = make(0.1).cuda().to(torch.bfloat16)
    opt = hvd.DistributedOptimizer(torch.optim.AdamW(m.parameters(), lr=1e-3),
                                   named_parameters=m.named_parameters())
    assert opt.fused_engine is not None
    x, y = batch()
    _no_sdpa(monkeypatch)

    def step(xb, yb):
        loss = F.cross_entropy(m(xb).float(), yb)
        loss.backward()
        opt.step()
        opt.zero_grad()
        return loss.detach()

    c0 = counters.snapshot()
    l0 = float(step(x, y))
    c1 = counters.snapshot()
    assert c1.get("attn_fwd_dropout", 0) - c0.get("attn_fwd_dropout", 0) == 2
    assert c1.get("attn_bwd_dropout", 0) > c0.get("attn_bwd_dropout", 0)
    assert c1.get("dropout_add", 0) - c0.get("dropout_add", 0) >= 2 * 2 * 2 + 1 + 1   # 4 branches fwd + bwd, input
    assert c1.get("attn_fwd", 0) == c0.get("attn_fwd", 0)
    graphed = GraphedStep(step, [x, y], warmup=2)
    losses = [float(graphed(x, y)) for _ in range(3)]
    torch.cuda.synchronize()
    print(f"\n[{name} dropout 0.1] eager loss {l0:.4f}, graphed {losses}")
    assert all(math.isfinite(v) for v in [l0] + losses)
    assert all(bool(torch.isfinite(p).all()) for p in m.parameters())


@gpu
@pytest.mark.parametrize("name", ["gpt", "vit"])
def test_eval_and_p0_match_the_model_without_dropout(name):
    from distributed_torch_horovod_gcp_b200.ops import functional as F2
    make, batch = _models()[name]
    torch.manual_seed(0)
    ref = make(0.0).cuda().to(torch.bfloat16)
    if name == "vit":
        torch.nn.init.normal_(ref.head.weight)             # the head starts at zero, which would hide any difference
    drop = make(0.1).cuda().to(torch.bfloat16)
    drop.load_state_dict(ref.state_dict())
    x, _ = batch()
    with torch.no_grad():
        ref.eval()
        drop.eval()
        assert torch.equal(drop(x), ref(x))
        # dropout 0 in training mode: the blocks run the calls they ran before dropout existed
        ref.train()
        got = ref(x)
        want = _forward_without_dropout(ref, x, F2)
        assert torch.equal(got, want)


def _block_without_dropout(blk, x, F2):
    h = F2.layer_norm(x, blk.ln_1.weight, blk.ln_1.bias, blk.ln_1.eps)
    a = F2.qkv_attention(h, blk.qkv.weight, blk.qkv.bias, blk.heads, blk.causal)
    x = F2.linear(a, blk.proj.weight, blk.proj.bias, residual=x)
    h = F2.layer_norm(x, blk.ln_2.weight, blk.ln_2.bias, blk.ln_2.eps)
    return F2.mlp(h, blk.fc1.weight, blk.fc1.bias, blk.fc2.weight, blk.fc2.bias, residual=x)


def _forward_without_dropout(m, x, F2):
    """The models' forward as written before they took a dropout argument."""
    if hasattr(m, "wte"):
        B, S = x.shape
        h = m.wte(x) + m.wpe.weight[:S]
        for blk in m.layers:
            h = _block_without_dropout(blk, h, F2)
        h = F2.layer_norm(h, m.ln_f.weight, m.ln_f.bias, m.ln_f.eps)
        return F2.linear(h.reshape(B * S, m.dim), m.wte.weight)
    B = x.shape[0]
    h = F2.patch_embed(x, m.conv_proj.weight, m.conv_proj.bias, m.patch)
    h = torch.cat([m.class_token.expand(B, -1, -1).to(h.dtype), h], dim=1)
    h = h + m.pos_embedding.to(h.dtype)
    for blk in m.layers:
        h = _block_without_dropout(blk, h, F2)
    h = F2.layer_norm(h[:, 0], m.ln.weight, m.ln.bias, m.ln.eps)
    return F2.linear(h, m.head.weight, m.head.bias)
