"""Sequence-parallel flash attention (csrc/attn_sm90.cu, ``SP = true``; ops/seq_parallel.py) at world sizes 1 to 8
on one GPU.

The kernels reach other ranks' data only through the gathered buffers they are given, so "rank r of W" runs
exactly on one GPU.  Each case builds the full-sequence q, k, v and dO, runs the existing full-sequence kernels
once as the reference, and for every emulated rank builds exactly what the op's collectives would deliver (the
op's own pack functions, stacked in rank order as the all-gather writes them), calls the new entry points and
checks:
- O, LSE, dK and dV against the reference rows bit for bit;
- dQ (the fp32 rank-order sum of every rank's partials, cast to bf16 by the op's cast kernel) within the float64
  bounds of the full-sequence kernel (``causal_bwd_bounds`` / ``attn_bwd_bounds``);
- every output lies in a buffer with NaN guard elements on both sides, which must be unchanged, and the host-side
  launch guard (``tests/launch_guard.py``, extended here with the new entry points) checks every pointer extent.
"""
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TESTS = os.path.dirname(os.path.abspath(__file__))
for _p in (ROOT, TESTS):
    if _p not in sys.path:
        sys.path.insert(0, _p)

import launch_guard  # noqa: E402
from fp64_bounds import assert_within_bound, report_ratios  # noqa: E402
from launch_guard import OPT, REQ, _span4  # noqa: E402
from test_gpu_causal_attention import causal_bwd_bounds  # noqa: E402
from test_gpu_vit_numerics import attn_bwd_bounds, attn_layout  # noqa: E402

gpu = pytest.mark.gpu
GUARD = 256


@pytest.fixture(scope="module", autouse=True)
def _report_ratios():
    yield
    report_ratios()


# ------------------------------------------------------------------ launch-guard entries of the new entry points
def _span5(a, st):
    """Elements spanned by a gathered [W, B, H, S, D] view with (rank, batch, head, seq) strides st."""
    if a.world <= 0 or a.B <= 0 or a.H <= 0 or a.S <= 0:
        return 0
    return (a.world - 1) * st[0] + (a.B - 1) * st[1] + (a.H - 1) * st[2] + (a.S - 1) * st[3] + a.D


def _rows(a):
    """Bytes of the gathered fp32 LSE or delta: rank stride ld_sw, B H S rows per rank."""
    return 4 * ((a.world - 1) * a.ld_sw + a.B * a.H * a.S)


SP_TABLE = {
    "b200dp_attn_delta": (("o", "do", "delta", "B", "H", "S", "D", "so", "sdo", "stream"), {
        "o": (lambda a: 2 * _span4(a, a.so, a.D), 16, REQ), "do": (lambda a: 2 * _span4(a, a.sdo, a.D), 16, REQ),
        "delta": (lambda a: 4 * a.B * a.H * a.S, 4, REQ),
    }),
    "b200dp_attn_sp_fwd": (("q", "k", "v", "o", "lse", "B", "H", "S", "D", "sq", "sk", "sv", "so", "scale", "causal",
                            "rank", "world", "stream"), {
        "q": (lambda a: 2 * _span4(a, a.sq, a.D), 16, REQ), "k": (lambda a: 2 * _span5(a, a.sk), 16, REQ),
        "v": (lambda a: 2 * _span5(a, a.sv), 16, REQ), "o": (lambda a: 2 * _span4(a, a.so, a.D), 16, REQ),
        "lse": (lambda a: 4 * a.B * a.H * a.S, 4, OPT),
    }),
    "b200dp_attn_sp_bwd": (("q", "k", "v", "do", "lse", "delta", "acc", "dk", "dv", "B", "H", "S", "D", "sq", "sk",
                            "sv", "sdo", "sacc", "sdk", "sdv", "ld_sw", "scale", "causal", "rank", "world", "stream"), {
        "q": (lambda a: 2 * _span5(a, a.sq), 16, REQ), "do": (lambda a: 2 * _span5(a, a.sdo), 16, REQ),
        "k": (lambda a: 2 * _span4(a, a.sk, a.D), 16, REQ), "v": (lambda a: 2 * _span4(a, a.sv, a.D), 16, REQ),
        "dk": (lambda a: 2 * _span4(a, a.sdk, a.D), 16, REQ), "dv": (lambda a: 2 * _span4(a, a.sdv, a.D), 16, REQ),
        "acc": (lambda a: 4 * _span5(a, a.sacc), 16, REQ),
        "lse": (_rows, 4, REQ), "delta": (_rows, 4, REQ),
    }),
}


@pytest.fixture
def guard(monkeypatch):
    _sp()                                                # loads the library, so its _lib is there to wrap
    for name, spec in SP_TABLE.items():
        monkeypatch.setitem(launch_guard.TABLE, name, spec)
    return launch_guard.install(monkeypatch)


def _sp():
    from distributed_torch_horovod_gcp_b200.ops import kernels, seq_parallel
    assert kernels.has("attention_fused"), "attention kernels missing from libb200dp_kernels.so"
    assert hasattr(seq_parallel._lib(), "b200dp_attn_sp_fwd"), "sequence-parallel entry points missing"
    return seq_parallel


# ------------------------------------------------------------------ guarded outputs
class Guarded:
    """A flat buffer of n elements between GUARD NaN elements on each side."""

    def __init__(self, n, dtype, fill=float("nan")):
        self.buf = torch.full((n + 2 * GUARD,), float("nan"), dtype=dtype, device="cuda")
        self.body = self.buf[GUARD:GUARD + n]
        self.body.fill_(fill)

    def check(self, what):
        assert bool(self.buf[:GUARD].isnan().all()) and bool(self.buf[-GUARD:].isnan().all()), \
            f"{what}: a guard element next to the output was written"
        assert not bool(self.body.isnan().any()), f"{what}: part of the output was never written"


def _bshd(g, B, H, S):
    """[B, H, S, 64] view of a [B, S, H, 64] memory buffer."""
    return g.body.view(B, S, H, 64).permute(0, 2, 1, 3)


# ------------------------------------------------------------------ reference: the full-sequence kernels
def _full_reference(q, k, v, do, causal):
    from distributed_torch_horovod_gcp_b200.ops import attention as A
    B, H, S, D = q.shape
    o = torch.empty((B, S, H, D), dtype=torch.bfloat16, device="cuda").permute(0, 2, 1, 3)
    lse = torch.empty((B, H, S), dtype=torch.float32, device="cuda")
    A._ck(A._lib.b200dp_attn_fwd_ex(q.data_ptr(), k.data_ptr(), v.data_ptr(), o.data_ptr(), lse.data_ptr(), B, H, S,
                                    D, A._strides(q), A._strides(k), A._strides(v), A._strides(o), 0.125, int(causal),
                                    torch.cuda.current_stream().cuda_stream))
    leaves = [t.clone().requires_grad_(True) for t in (q, k, v)]
    o2 = A.attention_fused(*leaves, causal=causal)
    o2.backward(do)
    torch.cuda.synchronize()
    assert torch.equal(o2.detach(), o)
    return o, lse, leaves[1].grad, leaves[2].grad


# (world, chunk tiles c, causal, B, H, layout of the local q / k / v / dO)
CASES = [
    (1, 1, True, 2, 1, "bshd"), (1, 2, False, 1, 2, "packed"),
    (2, 1, True, 1, 2, "bshd"), (2, 2, False, 2, 1, "bhsd"), (2, 3, True, 1, 2, "packed"),
    (3, 1, True, 1, 3, "packed"), (3, 2, True, 2, 1, "bshd"), (3, 1, False, 2, 1, "bshd"),
    (4, 1, False, 1, 2, "packed"), (4, 2, True, 1, 2, "bshd"),
    (8, 1, True, 2, 1, "bshd"), (8, 2, True, 1, 2, "packed"), (8, 1, False, 1, 2, "bhsd"),
]


@gpu
@pytest.mark.parametrize("W,c,causal,B,H,layout", CASES)
def test_emulated_ranks_bit_for_bit(W, c, causal, B, H, layout, guard):
    sp = _sp()
    S_loc = 2 * c * 128
    S = W * S_loc
    g = torch.Generator().manual_seed(1000 * W + 10 * c + int(causal))
    q, k, v, do = [torch.randn(B, H, S, 64, generator=g).bfloat16().cuda() for _ in range(4)]
    o_ref, lse_ref, dk_ref, dv_ref = _full_reference(q, k, v, do, causal)
    shard = (lambda t, r: sp.zigzag_shard(t, 2, r, W))
    local = [[attn_layout(shard(t, r), layout, slot % 3) for slot, t in enumerate((q, k, v, do))] for r in range(W)]
    n = B * S_loc * H * 64

    # ---- forward: the all-gather of every rank's packed K|V, then rank r's launch
    gathered_kv = torch.stack([sp.pack_kv(lk, lv) for _, lk, lv, _ in local])
    kg, vg = sp.kv_views(gathered_kv)
    outs = []
    for r in range(W):
        o, lse = Guarded(n, torch.bfloat16), Guarded(B * H * S_loc, torch.float32)
        sp.sp_fwd(local[r][0], kg, vg, _bshd(o, B, H, S_loc), lse.body.view(B, H, S_loc), causal, r, W)
        torch.cuda.synchronize()
        o.check(f"rank {r} O")
        lse.check(f"rank {r} LSE")
        assert torch.equal(_bshd(o, B, H, S_loc), shard(o_ref, r)), f"rank {r}: O differs from the full kernel's rows"
        assert torch.equal(lse.body.view(B, H, S_loc), shard(lse_ref, r)), f"rank {r}: LSE differs"
        outs.append((_bshd(o, B, H, S_loc), lse.body.view(B, H, S_loc)))
    assert guard["b200dp_attn_sp_fwd"] == W

    # ---- backward: every rank's Q|dO|LSE|delta pack gathered, then rank r's launch
    packs = [sp.pack_bwd(local[s][0], local[s][3], outs[s][0], outs[s][1]) for s in range(W)]
    gathered = torch.stack(packs)
    qg, dog, lse_ptr, delta_ptr, ld_sw = sp.bwd_views(gathered, B, H, S_loc)
    dq32 = torch.zeros((W, B, S_loc, H, 64), dtype=torch.float32, device="cuda")
    for r in range(W):
        acc = Guarded(W * n, torch.float32, fill=0.0)
        dk, dv = Guarded(n, torch.bfloat16), Guarded(n, torch.bfloat16)
        acc_v = acc.body.view(W, B, S_loc, H, 64)
        sp.sp_bwd(qg, local[r][1], local[r][2], dog, lse_ptr, delta_ptr, ld_sw, acc_v.permute(0, 1, 3, 2, 4),
                  _bshd(dk, B, H, S_loc), _bshd(dv, B, H, S_loc), causal, r, W)
        torch.cuda.synchronize()
        for name, t in (("dQ partials", acc), ("dK", dk), ("dV", dv)):
            t.check(f"rank {r} {name}")
        assert torch.equal(_bshd(dk, B, H, S_loc), shard(dk_ref, r)), f"rank {r}: dK differs from the full kernel's"
        assert torch.equal(_bshd(dv, B, H, S_loc), shard(dv_ref, r)), f"rank {r}: dV differs from the full kernel's"
        dq32 += acc_v                                    # the reduce-scatter's rank-order fp32 sum
    assert guard["b200dp_attn_sp_bwd"] == W and guard["b200dp_attn_delta"] == W
    dq_shards = []
    for s in range(W):
        out = Guarded(n, torch.bfloat16)
        sp.cast_bf16(dq32[s], out.body)
        torch.cuda.synchronize()
        out.check(f"rank {s} dQ")
        dq_shards.append(_bshd(out, B, H, S_loc))
    dq = sp.zigzag_unshard(dq_shards, 2)
    (dq64, dq_b), _, _ = (causal_bwd_bounds if causal else attn_bwd_bounds)(q, k, v, do, o_ref)
    assert_within_bound(dq, dq64, group=f"sp dq W={W}", terms=[(1.0, dq_b)])


class _OneRankSymm:
    """The collectives of a world of one: the all-gather and the reduce-scatter are copies."""

    def allgather(self, src, out):
        out.view(-1).copy_(src.reshape(-1))

    def reducescatter(self, src, out, scale=1.0):
        out.view(-1).copy_(src.reshape(-1))


@gpu
@pytest.mark.parametrize("causal", [True, False])
def test_op_world_one_matches_attention_fused(causal, guard):
    """The autograd Function with the collectives of a world of one against ``attention_fused``: O, dK, dV bit for
    bit, dQ within its bound; and ``sp_attention`` at world size 1 is ``attention_fused``."""
    sp = _sp()
    from distributed_torch_horovod_gcp_b200.ops import attention as A
    B, H, S = 2, 2, 512
    g = torch.Generator().manual_seed(7)
    q, k, v, do = [torch.randn(B, H, S, 64, generator=g).bfloat16().cuda() for _ in range(4)]
    ref = [t.clone().requires_grad_(True) for t in (q, k, v)]
    o_ref = A.attention_fused(*ref, causal=causal)
    o_ref.backward(do)
    mine = [attn_layout(t, "bshd").requires_grad_(True) for t in (q, k, v)]
    o = sp._SPAttnFn.apply(*mine, causal, 0, 1, _OneRankSymm())
    o.backward(do)
    torch.cuda.synchronize()
    assert torch.equal(o, o_ref) and o.stride() == o_ref.stride()
    assert torch.equal(mine[1].grad, ref[1].grad) and torch.equal(mine[2].grad, ref[2].grad)
    (dq64, dq_b), _, _ = (causal_bwd_bounds if causal else attn_bwd_bounds)(q, k, v, do, o_ref.detach())
    assert_within_bound(mine[0].grad, dq64, group="sp op dq (world 1)", terms=[(1.0, dq_b)])
    assert guard["b200dp_attn_sp_fwd"] == 1 and guard["b200dp_attn_sp_bwd"] == 1
    same = [t.detach().clone().requires_grad_(True) for t in (q, k, v)]
    o1 = sp.sp_attention(*same, causal=causal)
    assert torch.equal(o1, o_ref)


@gpu
def test_entry_points_refuse_bad_shapes():
    """A shard that is not a multiple of 256 rows, a rank outside the world, a wrong head dim: errors, no launch."""
    sp = _sp()
    from distributed_torch_horovod_gcp_b200.ops import attention as A
    q = torch.zeros(1, 1, 384, 64, dtype=torch.bfloat16, device="cuda")
    kg = torch.zeros(2, 1, 1, 384, 64, dtype=torch.bfloat16, device="cuda")
    o = torch.empty_like(q)
    for S, rank, world, D in ((384, 0, 2, 64), (256, 2, 2, 64), (256, 0, 2, 32)):
        with pytest.raises(RuntimeError):
            A._ck(A._lib.b200dp_attn_sp_fwd(q.data_ptr(), kg.data_ptr(), kg.data_ptr(), o.data_ptr(), None, 1, 1, S, D,
                                            A._strides(q), sp._strides4(kg), sp._strides4(kg), A._strides(o), 0.125, 1,
                                            rank, world, torch.cuda.current_stream().cuda_stream))


@gpu
@pytest.mark.multigpu
@pytest.mark.parametrize("causal", [True, False])
def test_multigpu_kernel_path_matches_single_gpu(causal):
    from mp_util import run_workers
    world = min(torch.cuda.device_count(), 8)
    assert all(run_workers(world, "sp_cases", "kernel_attention_matches_full", args=(2, 2, 512 * world, causal),
                           cuda=True, timeout=600))


@gpu
@pytest.mark.multigpu
def test_multigpu_gpt_step_matches_single_gpu():
    from mp_util import run_workers
    world = min(torch.cuda.device_count(), 8)
    res = run_workers(world, "sp_cases", "kernel_gpt_step", args=(2, 512 * world), cuda=True, timeout=600)
    assert len({r["loss"] for r in res}) == 1, res
