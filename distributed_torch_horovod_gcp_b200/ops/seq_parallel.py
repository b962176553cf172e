"""Sequence-parallel attention: every rank of the world holds a zigzag shard of each sequence, so the
activations, saved tensors and attention FLOPs of one sequence are split across the GPUs of a node.

Sharding (zigzag).  A global sequence of S positions is cut into 2W chunks of S / (2W); rank r holds chunks
r and 2W - 1 - r, in that order, as its S / W local rows (``zigzag_shard``, ``zigzag_positions``).  Under a
causal mask every rank then has the same number of (query, key) pairs to compute.

``sp_attention(q, k, v, causal=True)`` is attention of this rank's queries against the keys and values of the
whole sequence, an autograd Function over the local shard ([B, H, S_loc, 64] tensors, as
``attention.attention_fused`` takes them).  Kernel path (CUDA bf16, head dim 64, S_loc a multiple of 256, the
symmetric-memory runtime up):
- forward: one packed all-gather of K|V through ``runtime.symm`` (NVLink, no host round trip), then
  ``b200dp_attn_sp_fwd`` (csrc/attn_sm90.cu); only the local q, k, v, O and LSE are saved;
- backward: delta = rowsum(dO o O) on the local rows, one packed all-gather of Q|dO|LSE|delta,
  ``b200dp_attn_sp_bwd`` (dK, dV of the local keys over every rank's queries, dQ partials of every rank's
  queries into an fp32 [W, B, S_loc, H, 64] workspace), one fp32 reduce-scatter of that workspace and a cast
  to bf16.
O, LSE, dK and dV are bit-identical to the full-sequence kernels' rows; dQ differs only in the order of its
fp32 sums.  Anywhere else (CPU / Gloo, other dtypes, head dims or lengths) the reference path runs: a
differentiable ``torch.distributed`` all-gather of K and V and SDPA with a boolean mask built from the global
positions.  At world size 1, ``sp_attention`` is ``attention_fused`` (or SDPA where the kernels do not apply).

Groups.  ``sp_attention(..., process_set=ps)`` splits each sequence across the ranks of ``ps`` only: "rank" and
"world" above are then the rank's index in the set and the set's size, the all-gathers and the reduce-scatter run
among the set's members (``runtime.symm`` with ``members=``, never multicast) and the reference path uses the
set's ``torch.distributed`` group.  Several disjoint sets (``models.gpt``: contiguous blocks of ranks) then train
on different batches at once.  A set of one rank is plain attention; a set of the whole world is the world.

Not supported: attention dropout (the backward would need each query row owner's Philox seed), CUDA-graph capture
of the kernel path (its collectives are launched with per-call host arguments)."""
from __future__ import annotations

import ctypes
import logging
import math

import torch
import torch.distributed as dist
import torch.nn.functional as F

from .. import _state
from . import attention as _attn
from . import counters

log = logging.getLogger("b200dp")
TILE = 128
_said = set()


# ------------------------------------------------------------------ zigzag helpers
def _chunk(S: int, world: int) -> int:
    if world < 1 or S % (2 * world):
        raise ValueError(f"a sequence of {S} positions does not split into 2 x {world} equal zigzag chunks")
    return S // (2 * world)


def zigzag_positions(S: int, rank: int, world: int, device=None) -> torch.Tensor:
    """Global positions (int64) of the S / world local rows of ``rank``: chunks rank and 2 world - 1 - rank."""
    L = _chunk(S, world)
    a = torch.arange(L, device=device, dtype=torch.int64)
    return torch.cat([a + rank * L, a + (2 * world - 1 - rank) * L])


def zigzag_shard(x: torch.Tensor, dim: int, rank: int, world: int) -> torch.Tensor:
    """Rank ``rank``'s zigzag shard of ``x`` along ``dim`` (a new tensor)."""
    L = _chunk(x.shape[dim], world)
    return torch.cat([x.narrow(dim, rank * L, L), x.narrow(dim, (2 * world - 1 - rank) * L, L)], dim)


def zigzag_unshard(shards, dim: int) -> torch.Tensor:
    """The full tensor from every rank's shard (``shards[r]`` = rank r's), along ``dim``."""
    L = shards[0].shape[dim] // 2
    first = [s.narrow(dim, 0, L) for s in shards]
    second = [s.narrow(dim, L, L) for s in reversed(shards)]
    return torch.cat(first + second, dim)


# ------------------------------------------------------------------ kernel path
def _lib():
    return _attn._lib


def _strides4(t):
    """(rank, batch, head, seq) element strides of a gathered [W, B, H, S, D] view."""
    return (ctypes.c_longlong * 4)(*t.stride()[:4])


def pack_kv(k, v) -> torch.Tensor:
    """This rank's K|V as one contiguous [2, B, S, H, 64] bf16 buffer: the all-gather's input."""
    B, H, S, D = k.shape
    kv = torch.empty((2, B, S, H, D), dtype=torch.bfloat16, device=k.device)
    kv[0].copy_(k.transpose(1, 2))
    kv[1].copy_(v.transpose(1, 2))
    return kv


def kv_views(g: torch.Tensor):
    """The gathered K and V ([W, B, H, S, 64] views) of the all-gather of every rank's ``pack_kv``
    (``g``: [W, 2, B, S, H, 64] in rank order)."""
    return g[:, 0].permute(0, 1, 3, 2, 4), g[:, 1].permute(0, 1, 3, 2, 4)


def bwd_pack_layout(B, H, S, D=64):
    """Byte offsets of Q, dO, LSE and delta in one rank's backward pack, and its size."""
    nq = B * S * H * D * 2
    nl = B * H * S * 4
    return (0, nq, 2 * nq, 2 * nq + nl), 2 * nq + 2 * nl


def pack_bwd(q, do, o, lse) -> torch.Tensor:
    """This rank's Q|dO|LSE|delta as one uint8 buffer (delta = rowsum(dO o O) computed here): the backward
    all-gather's input."""
    B, H, S, D = q.shape
    (oq, od, ol, oe), n = bwd_pack_layout(B, H, S, D)
    buf = torch.empty(n, dtype=torch.uint8, device=q.device)
    buf[oq:od].view(torch.bfloat16).view(B, S, H, D).copy_(q.transpose(1, 2))
    buf[od:ol].view(torch.bfloat16).view(B, S, H, D).copy_(do.transpose(1, 2))
    buf[ol:oe].view(torch.float32).view(B, H, S).copy_(lse)
    delta = buf[oe:].view(torch.float32)
    _attn._ck(_lib().b200dp_attn_delta(o.data_ptr(), do.data_ptr(), delta.data_ptr(), B, H, S, D, _attn._strides(o),
                                       _attn._strides(do), torch.cuda.current_stream(q.device).cuda_stream))
    return buf


def bwd_views(g: torch.Tensor, B, H, S, D=64):
    """Gathered Q, dO ([W, B, H, S, 64] views), the LSE and delta base pointers and their rank stride (fp32
    elements) of the all-gather ``g`` ([W, n] uint8, rank order) of every rank's ``pack_bwd``."""
    W = g.shape[0]
    (oq, od, ol, oe), n = bwd_pack_layout(B, H, S, D)
    qg = g[:, oq:od].view(torch.bfloat16).view(W, B, S, H, D).permute(0, 1, 3, 2, 4)
    dog = g[:, od:ol].view(torch.bfloat16).view(W, B, S, H, D).permute(0, 1, 3, 2, 4)
    return qg, dog, g.data_ptr() + ol, g.data_ptr() + oe, n // 4


def sp_fwd(q, kg, vg, o, lse, causal: bool, rank: int, world: int):
    """``b200dp_attn_sp_fwd``: rank ``rank``'s O (and LSE unless None) from its Q and the gathered K, V."""
    B, H, S, D = q.shape
    _attn._ck(_lib().b200dp_attn_sp_fwd(
        q.data_ptr(), kg.data_ptr(), vg.data_ptr(), o.data_ptr(), lse.data_ptr() if lse is not None else None,
        B, H, S, D, _attn._strides(q), _strides4(kg), _strides4(vg), _attn._strides(o), 1.0 / math.sqrt(D),
        int(causal), rank, world, torch.cuda.current_stream(q.device).cuda_stream))


def sp_bwd(qg, k, v, dog, lse_ptr, delta_ptr, ld_sw, acc, dk, dv, causal: bool, rank: int, world: int):
    """``b200dp_attn_sp_bwd``: rank ``rank``'s dK, dV and its dQ partials of every rank's queries, added into
    ``acc`` ([W, B, H, S, 64] fp32 view, zero on entry)."""
    B, H, S, D = k.shape
    _attn._ck(_lib().b200dp_attn_sp_bwd(
        qg.data_ptr(), k.data_ptr(), v.data_ptr(), dog.data_ptr(), lse_ptr, delta_ptr, acc.data_ptr(), dk.data_ptr(),
        dv.data_ptr(), B, H, S, D, _strides4(qg), _attn._strides(k), _attn._strides(v), _strides4(dog), _strides4(acc),
        _attn._strides(dk), _attn._strides(dv), ld_sw, 1.0 / math.sqrt(D), int(causal), rank, world,
        torch.cuda.current_stream(k.device).cuda_stream))


def cast_bf16(src32: torch.Tensor, out: torch.Tensor):
    """``out`` (bf16, contiguous memory) = ``src32`` (fp32, same element order) on the cast kernel."""
    rc = _lib().b200dp_cast_acc_zero(src32.data_ptr(), out.data_ptr(), src32.numel(), 1, 0, 0,
                                     torch.cuda.current_stream(src32.device).cuda_stream)
    if rc != 0:
        raise RuntimeError("cast_acc_zero failed")


class _SPAttnFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, q, k, v, causal, rank, world, symm, members=None):
        q, k, v = _attn._fix(q), _attn._fix(k), _attn._fix(v)
        B, H, S, D = q.shape
        dev = q.device
        coll = {} if members is None else {"members": members}     # the group's ranks (world ranks), or the world
        g = torch.empty((world, 2, B, S, H, D), dtype=torch.bfloat16, device=dev)
        symm.allgather(pack_kv(k, v), g, **coll)
        kg, vg = kv_views(g)
        o = torch.empty((B, S, H, D), dtype=torch.bfloat16, device=dev).permute(0, 2, 1, 3)
        lse = torch.empty((B, H, S), dtype=torch.float32, device=dev)
        sp_fwd(q, kg, vg, o, lse, causal, rank, world)
        counters.bump("attn_sp_fwd")
        ctx.save_for_backward(q, k, v, o, lse)
        ctx.causal, ctx.rank, ctx.world, ctx.symm, ctx.coll = causal, rank, world, symm, coll
        return o

    @staticmethod
    def backward(ctx, do):
        q, k, v, o, lse = ctx.saved_tensors
        B, H, S, D = q.shape
        W, dev = ctx.world, q.device
        do = _attn._fix(do)
        pack = pack_bwd(q, do, o, lse)
        g = torch.empty((W, pack.numel()), dtype=torch.uint8, device=dev)
        ctx.symm.allgather(pack, g, **ctx.coll)
        qg, dog, lse_ptr, delta_ptr, ld_sw = bwd_views(g, B, H, S, D)
        acc = torch.zeros((W, B, S, H, D), dtype=torch.float32, device=dev)
        dk, dv = [torch.empty((B, S, H, D), dtype=torch.bfloat16, device=dev).permute(0, 2, 1, 3) for _ in range(2)]
        sp_bwd(qg, k, v, dog, lse_ptr, delta_ptr, ld_sw, acc.permute(0, 1, 3, 2, 4), dk, dv, ctx.causal, ctx.rank, W)
        dq32 = torch.empty((B, S, H, D), dtype=torch.float32, device=dev)
        ctx.symm.reducescatter(acc, dq32, **ctx.coll)      # rank r: sum over ranks of acc[r]
        dq = torch.empty((B, S, H, D), dtype=torch.bfloat16, device=dev)
        cast_bf16(dq32, dq)
        counters.bump("attn_sp_bwd", 3)
        return dq.permute(0, 2, 1, 3), dk, dv, None, None, None, None, None


# ------------------------------------------------------------------ reference path
class _GatherSeq(torch.autograd.Function):
    """All-gather of [B, H, S, D] shards along S in rank order; the backward sums the full gradient over ranks
    and returns this rank's rows."""

    @staticmethod
    def forward(ctx, x, rank, world, group):
        x = x.contiguous()
        outs = [torch.empty_like(x) for _ in range(world)]
        dist.all_gather(outs, x, group=group)
        ctx.rank, ctx.S, ctx.group = rank, x.shape[2], group
        return torch.cat(outs, dim=2)

    @staticmethod
    def backward(ctx, g):
        g = g.contiguous()
        dist.all_reduce(g, group=ctx.group)
        return g.narrow(2, ctx.rank * ctx.S, ctx.S), None, None, None


def sp_attention_reference(q, k, v, causal: bool, rank: int, world: int, group=None):
    """The kernel path's result composed from torch: gathered K, V and SDPA with a mask on global positions."""
    S_loc = q.shape[2]
    if S_loc % 2:
        raise ValueError(f"a zigzag shard has an even number of rows, got {S_loc}")
    if group is None:
        from ..torch.mpi_ops import _group_for
        group = _group_for(q)
    kf = _GatherSeq.apply(k, rank, world, group)
    vf = _GatherSeq.apply(v, rank, world, group)
    mask = None
    if causal:
        S = S_loc * world
        pq = zigzag_positions(S, rank, world, q.device)
        pk = torch.cat([zigzag_positions(S, r, world, q.device) for r in range(world)])
        mask = pk[None, :] <= pq[:, None]
    return F.scaled_dot_product_attention(q, kf, vf, attn_mask=mask)


# ------------------------------------------------------------------ dispatch
def _kernel_reason(q, k, v):
    """None where the kernel path applies, else why not."""
    if _lib() is None or not hasattr(_lib(), "b200dp_attn_sp_fwd"):
        return "the attention kernels are not built"
    if not q.is_cuda:
        return "tensors are not on a GPU"
    if not _attn.supported(q, k, v):
        return "the kernels take bf16 [B, H, S, 64] q, k, v of one shape with 16-byte aligned rows"
    if q.shape[2] % (2 * TILE):
        return f"the local sequence ({q.shape[2]}) is not a multiple of {2 * TILE}"
    return None


def _split(process_set):
    """(rank, world, members, torch.distributed group) of the sequence split: this rank of the whole world
    (members and group None), or its index in ``process_set`` and the set's size, world ranks and group."""
    rt = _state.runtime()
    rank, world = (rt.rank, rt.size) if rt.initialized else (0, 1)
    if process_set is None or world == 1 or process_set.size() == world:
        return rank, world, None, None
    return process_set.rank(), process_set.size(), list(process_set.ranks), process_set.group


def sp_attention(q, k, v, causal: bool = True, dropout_p: float = 0.0, process_set=None):
    """softmax(q k^T / sqrt(d) [+ causal mask on global positions]) v for this rank's zigzag shard of the
    queries against every rank's keys and values: q, k, v are [B, H, S_loc, d] shards (see the module
    docstring); returns [B, H, S_loc, d] (kernel path: memory order [B, S_loc, H, d]).  ``process_set``: split
    across the ranks of this ``hvd.ProcessSet`` only (None: the world).  ``dropout_p > 0`` is only supported
    when the split has one rank."""
    dropout_p = _attn.check_dropout_p(dropout_p)
    rank, world, members, group = _split(process_set)
    if world == 1:
        if _attn._lib is not None and q.is_cuda and _attn.supported(q, k, v):
            return _attn.attention_fused(q, k, v, causal, dropout_p)
        return F.scaled_dot_product_attention(q, k, v, dropout_p=dropout_p, is_causal=causal)
    if dropout_p > 0.0:
        raise ValueError("attention dropout is not supported under sequence parallelism")
    if not (q.shape == k.shape == v.shape):
        raise ValueError(f"sequence-parallel attention needs q, k, v of one shape, got "
                         f"{tuple(q.shape)}, {tuple(k.shape)}, {tuple(v.shape)}")
    why = _kernel_reason(q, k, v)
    symm = None
    if why is None:
        if torch.cuda.is_current_stream_capturing():
            raise RuntimeError("sequence-parallel attention cannot be captured in a CUDA graph: its collectives "
                               "are launched with per-call host arguments")
        symm = _state.get_symm(q.device)
        if symm is None:
            why = "the symmetric-memory runtime is unavailable"
    if why is None:
        return _SPAttnFn.apply(q, k, v, bool(causal), rank, world, symm, members)
    if why not in _said:
        _said.add(why)
        log.warning("sp_attention: reference path (all-gather + SDPA with a mask) because %s", why)
    return sp_attention_reference(q, k, v, bool(causal), rank, world, group)
