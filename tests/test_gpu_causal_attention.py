"""Causal flash attention (csrc/attn_sm90.cu, ``CAUSAL = true``) and the GPT model on it.

1. Forward (O and LSE) and backward (dQ, dK, dV) against float64 causal attention, element by element, with
   bounds derived as in ``test_gpu_vit_numerics`` (``attn_fwd_bounds`` / ``attn_bwd_bounds``) but summed over
   the unmasked keys only: the kernel's masked products are exact zeros, so they add neither value nor error.
2. The non-causal kernel's O, dK and dV bit for bit against digests recorded before the causal mask existed.
3. The mask's edges exactly: row 0 is v's row 0, rows before t ignore k / v at t and after, and keys whose
   every query has a zero output gradient get exactly zero dK / dV.
4. GPT-2 small and gpt_tiny on the kernel path: no SDPA call, agreement with the cuBLAS + SDPA path, exact
   causality of the logits, and a fused-engine training step, eager and CUDA-graphed.

Run as a script on an H100 (``python tests/test_gpu_causal_attention.py``) to print the SHA-256 digests of
the non-causal kernel's outputs that ``tests/golden/attention_noncausal_sha256.json`` pins.
"""
import hashlib
import json
import math
import os
import sys

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

GOLDEN = os.path.join(TESTS, "golden", "attention_noncausal_sha256.json")
TILE = 128
CAUSAL_S = [1, 2, 63, 64, 65, 127, 128, 129, 255, 256, 257, 1024, 2048]


@pytest.fixture(scope="module", autouse=True)
def _report_ratios():
    yield
    report_ratios()


def _t(x):
    return x.transpose(-1, -2)


def _sha(t):
    return hashlib.sha256(t.detach().contiguous().cpu().view(torch.int16).numpy().tobytes()).hexdigest()


def _attn():
    from distributed_torch_horovod_gcp_b200.ops import attention, kernels
    assert kernels.has("attention_fused"), "attention kernels missing from libb200dp_kernels.so"
    return attention


# ================================================================================================ references
def _future(S, device):
    """[S, S] True where key j > query i (masked)."""
    return torch.ones(S, S, dtype=torch.bool, device=device).triu(1)


def causal_ref64(q, k, v):
    """float64 causal softmax(q k^T / 8) v and the natural-log LSE over the unmasked scores."""
    q, k, v = q.double(), k.double(), v.double()
    s = (q @ _t(k) / 8.0).masked_fill(_future(q.shape[2], q.device), float("-inf"))
    lse = torch.logsumexp(s, dim=-1)
    return torch.exp(s - lse[..., None]) @ v, lse


def causal_fwd_bounds(q, k, v):
    """``attn_fwd_bounds`` of test_gpu_vit_numerics with every row's maxima, minima, exponent errors and
    P* |V| sums taken over its unmasked keys 0..i.  The accumulation terms keep S and nb = ceil(S / 128),
    upper bounds of the keys and KV blocks any row visits."""
    q, k, v = q.detach(), k.detach(), v.detach()
    q64, k64, v64 = q.double(), k.double(), v.double()
    S = q.shape[2]
    nb = -(-S // TILE)
    fut = _future(S, q.device)
    o, lse = causal_ref64(q, k, v)
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
    phi = (1 + eps_l / (1 - eps_l)) * (1 + U_DIV) * (1 + U32) - 1
    c_z = w + (U_BF16 + eps_acc * (1 + U_BF16)) * (1 + w) + phi * (1 + w) * (1 + U_BF16) * (1 + eps_acc)
    o_terms = [((1 + U_BF16) * c_z, p @ v64.abs()), (U_BF16, o.abs())]
    c_lse = LN2 * (-torch.log2(1 - eta) - math.log2(1 - eps_l) + U_LOG2 * (math.log2(S) + 1)) * (1 + 4 * U32)
    c_lse = c_lse.squeeze(-1)
    lse_terms = [(c_lse, torch.ones_like(lse)), (4 * U32, lse.abs())]
    lse_bound = c_lse + 4 * U32 * lse.abs()
    return o, lse, o_terms, lse_terms, lse_bound


def causal_bwd_bounds(q, k, v, do, o_k):
    """``attn_bwd_bounds`` of test_gpu_vit_numerics with P*, its error and dS zero at masked (query, key)
    pairs, where the kernel's P and dS are exact zeros."""
    q64, k64, v64 = [t.detach().double().requires_grad_(True) for t in (q, k, v)]
    do64 = do.double()
    o, lse = causal_ref64(q64, k64, v64)
    o.backward(do64)
    dq, dk, dv = q64.grad, k64.grad, v64.grad
    q64, k64, v64, o, lse = q64.detach(), k64.detach(), v64.detach(), o.detach(), lse.detach()
    S = q.shape[2]
    nb = -(-S // TILE)
    keep = ~_future(S, q.device)
    _, _, _, _, lse_bound = causal_fwd_bounds(q, k, v)
    s = q64 @ _t(k64) / 8.0
    P = torch.exp(s - lse[..., None]) * keep
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


# ================================================================================================ kernel calls
def _causal_fwd(q, k, v):
    """``b200dp_attn_fwd_ex(causal = 1)`` called directly, with an LSE buffer; o in [B, S, H, 64] order."""
    A = _attn()
    B, H, S, D = q.shape
    o = torch.full((B, S, H, D), float("nan"), dtype=torch.bfloat16, device="cuda").permute(0, 2, 1, 3)
    lse = torch.full((B, H, S), float("nan"), dtype=torch.float32, device="cuda")
    A._ck(A._lib.b200dp_attn_fwd_ex(q.data_ptr(), k.data_ptr(), v.data_ptr(), o.data_ptr(), lse.data_ptr(),
                                    B, H, S, D, A._strides(q), A._strides(k), A._strides(v), A._strides(o), 0.125,
                                    1, torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    return o, lse


def _causal_fwd_bwd(q, k, v, do, layout):
    """``attention_fused(causal=True)`` forward + backward with q, k, v and dO in ``layout``."""
    A = _attn()
    leaves = [attn_layout(t.detach(), layout, slot).requires_grad_(True) for slot, t in enumerate((q, k, v))]
    o = A.attention_fused(*leaves, causal=True)
    o.backward(attn_layout(do, layout))
    torch.cuda.synchronize()
    return o.detach(), [t.grad for t in leaves]


def _workspace_zero():
    return all(float(w.abs().max()) == 0.0 for w in _attn()._ws.values())


# ================================================================================================ numerics
@gpu
@pytest.mark.parametrize("layout", ["bhsd", "bshd"])
@pytest.mark.parametrize("S", CAUSAL_S)
def test_causal_fwd_vs_fp64(S, layout):
    q, k, v = [t.cuda() for t in attn_inputs(S, "plain", seed=S)]
    o, lse = _causal_fwd(*[attn_layout(t, layout) for t in (q, k, v)])
    o64, lse64, o_terms, lse_terms, _ = causal_fwd_bounds(q, k, v)
    assert_within_bound(o, o64, group=f"causal fwd o ({layout})", terms=o_terms)
    assert_within_bound(lse, lse64, group=f"causal fwd lse ({layout})", terms=lse_terms)


@gpu
@pytest.mark.parametrize("layout", ["bhsd", "bshd"])
@pytest.mark.parametrize("S", CAUSAL_S)
def test_causal_bwd_vs_fp64(S, layout):
    q, k, v = [t.cuda() for t in attn_inputs(S, "plain", seed=S + 7)]
    do = torch.randn(q.shape, generator=torch.Generator().manual_seed(S)).bfloat16().cuda()
    o, grads = _causal_fwd_bwd(q, k, v, do, layout)
    assert _workspace_zero(), "the dQ workspace was left non-zero"
    bounds = causal_bwd_bounds(q, k, v, do, o)
    for name, got, (ref, b) in zip(("dq", "dk", "dv"), grads, bounds):
        assert_within_bound(got, ref, group=f"causal bwd {name} ({layout})", terms=[(1.0, b)])
    # a second call on the same inputs: dK / dV are fixed-order sums (bit for bit), dQ is summed by fp32 atomics
    # in any order, so it agrees to its bound; a dQ workspace left dirty by the first call would double it
    o2, grads2 = _causal_fwd_bwd(q, k, v, do, layout)
    assert torch.equal(o2, o)
    assert torch.equal(grads2[1], grads[1]) and torch.equal(grads2[2], grads[2])
    assert_within_bound(grads2[0], bounds[0][0], group=f"causal bwd dq, 2nd call ({layout})",
                        terms=[(1.0, bounds[0][1])])


# ================================================================================================ non-causal bits
def noncausal_digests():
    """O, dK, dV of a seeded non-causal ``attention_fused`` call at S = 197 and 1024 (dQ is left out: the
    order of its fp32 RED.ADDs is not fixed)."""
    attention = _attn()
    out = {}
    for S in (197, 1024):
        g = torch.Generator().manual_seed(S)
        q, k, v, do = [torch.randn(2, 3, S, 64, generator=g).bfloat16().cuda() for _ in range(4)]
        q, k, v = [t.requires_grad_(True) for t in (q, k, v)]
        o = attention.attention_fused(q, k, v)
        o.backward(do)
        torch.cuda.synchronize()
        for name, t in (("o", o), ("dk", k.grad), ("dv", v.grad)):
            out[f"S{S}_{name}"] = _sha(t)
    return out


@gpu
def test_noncausal_bits_unchanged():
    with open(GOLDEN) as f:
        want = json.load(f)
    assert noncausal_digests() == want


# ================================================================================================ exact edges
@gpu
@pytest.mark.parametrize("S", [1, 129, 300])
def test_causal_row0_is_v0(S):
    q, k, v = [t.cuda() for t in attn_inputs(S, "plain", seed=3 * S)]
    o, _ = _causal_fwd(q, k, v)
    assert torch.equal(o[:, :, 0], v[:, :, 0])


@gpu
@pytest.mark.parametrize("t", [1, 77, 128, 200, 256])
def test_causal_future_keys_do_not_reach_earlier_rows(t):
    S = 300
    q, k, v = [t_.cuda() for t_ in attn_inputs(S, "plain", seed=11)]
    k2, v2 = k.clone(), v.clone()
    g = torch.Generator().manual_seed(t)
    k2[:, :, t:] = (4 * torch.randn(k2[:, :, t:].shape, generator=g)).bfloat16().cuda()
    v2[:, :, t:] = (4 * torch.randn(v2[:, :, t:].shape, generator=g)).bfloat16().cuda()
    o, _ = _causal_fwd(*[attn_layout(x, "bshd") for x in (q, k, v)])
    o2, _ = _causal_fwd(*[attn_layout(x, "bshd") for x in (q, k2, v2)])
    assert torch.equal(o2[:, :, :t], o[:, :, :t])
    assert not torch.equal(o2[:, :, t:], o[:, :, t:])


@gpu
@pytest.mark.parametrize("t0", [1, 77, 128, 250])
def test_causal_keys_after_the_last_gradient_get_none(t0):
    S = 300
    q, k, v = [t.cuda() for t in attn_inputs(S, "plain", seed=13)]
    do = torch.randn(q.shape, generator=torch.Generator().manual_seed(t0)).bfloat16().cuda()
    do[:, :, t0:] = 0
    _, (dq, dk, dv) = _causal_fwd_bwd(q, k, v, do, "bhsd")
    assert float(dk[:, :, t0:].abs().max()) == 0.0 and float(dv[:, :, t0:].abs().max()) == 0.0
    assert float(dv[:, :, :t0].abs().max()) > 0.0
    assert float(dq[:, :, t0:].abs().max()) == 0.0


@gpu
def test_causal_rejects_mismatched_lengths():
    A = _attn()
    q = torch.zeros(1, 1, 64, 64, dtype=torch.bfloat16, device="cuda")
    k = torch.zeros(1, 1, 128, 64, dtype=torch.bfloat16, device="cuda")
    with pytest.raises(ValueError):
        A.attention_fused(q, k, k, causal=True)


# ================================================================================================ GPT
def _rel(a, b):
    a, b = a.detach().double(), b.detach().double()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


@gpu
def test_gpt2_small_runs_on_the_causal_kernel(monkeypatch):
    """GPT-2 small, bf16, B = 2, S = 1024: every attention runs on the kernel (an SDPA call raises), logits and
    loss agree with the cuBLAS + SDPA path, and logits before a changed token are bit for bit unchanged."""
    import torch.nn.functional as F
    from distributed_torch_horovod_gcp_b200.models import gpt2
    from distributed_torch_horovod_gcp_b200.ops import counters
    _attn()
    torch.manual_seed(0)
    m = gpt2().cuda().to(torch.bfloat16)
    B, S = 2, 1024
    g = torch.Generator(device="cuda").manual_seed(1)
    idx = torch.randint(0, 50257, (B, S + 1), generator=g, device="cuda")
    x, y = idx[:, :-1], idx[:, 1:].reshape(-1)

    monkeypatch.setenv("B200DP_DISABLE_KERNELS", "1")
    with torch.no_grad():
        ref = m(x)
        ref_loss = F.cross_entropy(ref.float(), y)
    monkeypatch.delenv("B200DP_DISABLE_KERNELS")

    def _no_sdpa(*a, **kw):
        raise AssertionError("F.scaled_dot_product_attention was called on the kernel path")
    monkeypatch.setattr(F, "scaled_dot_product_attention", _no_sdpa)
    c0 = counters.snapshot()
    logits = m(x)
    loss = F.cross_entropy(logits.float(), y)
    loss.backward()
    torch.cuda.synchronize()
    c1 = counters.snapshot()
    assert c1.get("attn_fwd", 0) - c0.get("attn_fwd", 0) == 12
    assert c1.get("attn_bwd", 0) > c0.get("attn_bwd", 0)
    assert logits.shape == (B * S, 50304) and logits.dtype == torch.bfloat16
    e = _rel(logits, ref)
    print(f"\n[gpt2] logits rel err kernel vs stand-in {e:.3e}, loss {float(loss):.5f} vs {float(ref_loss):.5f}")
    assert e < 2e-2
    assert abs(float(loss) - float(ref_loss)) < 1e-2
    assert all(p.grad is not None and bool(torch.isfinite(p.grad).all()) for p in m.parameters())

    with torch.no_grad():
        base = m(x).view(B, S, -1)
        for t in (300, 512):
            alt = x.clone()
            alt[:, t:] = torch.randint(0, 50257, (B, S - t), generator=g, device="cuda")
            out = m(alt).view(B, S, -1)
            assert torch.equal(out[:, :t], base[:, :t]), f"logits before position {t} changed"


@gpu
def test_gpt_tiny_fused_adamw_step(hvd_single, monkeypatch):
    """gpt_tiny through hvd.DistributedOptimizer(AdamW) on the fused engine: the loss on a fixed batch falls
    over 20 steps, and a CUDA-graphed step replays with the loss of an eager forward on the same parameters."""
    import torch.nn.functional as F
    from distributed_torch_horovod_gcp_b200.models import gpt_tiny
    from distributed_torch_horovod_gcp_b200.utils.graph import GraphedStep
    monkeypatch.setenv("B200DP_FUSED_SINGLE", "1")
    hvd = hvd_single
    _attn()
    torch.manual_seed(0)
    m = gpt_tiny().cuda().to(torch.bfloat16)
    groups = [{"params": [p for p in m.parameters() if p.dim() >= 2], "weight_decay": 0.1},
              {"params": [p for p in m.parameters() if p.dim() < 2], "weight_decay": 0.0}]
    opt = hvd.DistributedOptimizer(torch.optim.AdamW(groups, lr=1e-3, betas=(0.9, 0.95)),
                                   named_parameters=m.named_parameters())
    assert opt.fused_engine is not None
    g = torch.Generator(device="cuda").manual_seed(2)
    x = torch.randint(0, 512, (4, 128), generator=g, device="cuda")
    y = torch.randint(0, 512, (4 * 128,), generator=g, device="cuda")

    def step(xb, yb):
        loss = F.cross_entropy(m(xb).float(), yb)
        loss.backward()
        opt.step()
        opt.zero_grad()
        return loss.detach()

    losses = [float(step(x, y)) for _ in range(20)]
    print(f"\n[gpt_tiny] losses {losses[0]:.4f} -> {losses[-1]:.4f}")
    assert all(math.isfinite(v) for v in losses)
    assert losses[-1] < losses[0] - 1.0
    graphed = GraphedStep(step, [x, y], warmup=2)
    with torch.no_grad():
        le = F.cross_entropy(m(x).float(), y)
    lg = graphed(x, y)
    torch.cuda.synchronize()
    torch.testing.assert_close(lg, le, rtol=1e-6, atol=0)


if __name__ == "__main__":
    print(json.dumps(noncausal_digests(), indent=1, sort_keys=True))
