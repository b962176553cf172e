"""The group forms of the reduce-scatter and all-gather kernels (``b200dp_comm_group_collective``) at world sizes 2,
4 and 8 and every group size 2 <= G <= W that divides W, every emulated rank of every group, on one GPU.

The emulation is ``test_gpu_comm_numerics``'s: one process runs "world rank r" exactly, through per-rank
``CommCtx`` blocks over N signal pads, one rank at a time from the same start state.  Here only the members of the
group are credited; the other ranks' pad entries are set to their epochs (never credited), so a kernel that waited
on a non-member would not finish.  Groups are the contiguous blocks [k G, (k + 1) G); data pointers are indexed by
group rank, and the argument block comes from ``runtime.symm.group_coll_args``, as the runtime builds it.

Checks:
- all-gather: slot g of every member's output holds member g's input, bit for bit;
- reduce-scatter: member g's output is the fp32 sum from +0 over the members' chunk g in group-rank order, times
  the scale, rounded once to the output type, bit for bit, and within the float64 bound of ``sum_bound``;
- write sets: every change lies in a member's own output (reduce-scatter) or the members' outputs (all-gather);
  every other rank's buffers and every guard element stay bit-unchanged;
- barrier bookkeeping: a rank adds 2 exactly to the pad entry [ch][b][r] of each other member and to its own epoch
  entry [ch][b][member] (world-rank indices), and to no other entry; the mailbox stays zero;
- one member left uncredited, with the mailbox already set: a watchdog exit that writes nothing.
"""
import ctypes
import zlib

import pytest
import torch

from test_gpu_comm_numerics import (BF16, BLOCKS, CH_USER, CHANNELS, DT_CODE, F16, F32, RANKS, THREADS, VN, Emu,
                                    _buf, _stream, check_sum, fp32, make_grads, owned_by, pattern)
from test_gpu_optimizer_numerics import Checker

gpu = pytest.mark.gpu

WG = [(W, G) for W in (2, 4, 8) for G in range(2, W + 1) if W % G == 0]


class GroupEmu(Emu):
    """``Emu`` whose launches are those of one group: non-members are not launched, only members are credited."""

    members = ()

    def launch(self, ck, tag, r, fn, ch, grid, uncredited=None):
        if r not in self.members:
            return
        pad = self.pads[r].view(CHANNELS, BLOCKS, RANKS)
        ep = self.epochs[r].view(CHANNELS, BLOCKS, RANKS)
        for t in range(self.N):
            if t != r:
                credit = 2 if t in self.members and t != uncredited else 0
                pad[ch, :grid, t] = ep[ch, :grid, t] + credit
        p0, e0 = self.pads.clone(), self.epochs.clone()
        rc = fn(self.ctx[r])
        assert rc == 0, self.lib.b200dp_comm_last_error()
        torch.cuda.synchronize()
        inc = 2 if uncredited is None else 1
        for t in self.members:
            if t != r:
                p0[t].view(CHANNELS, BLOCKS, RANKS)[ch, :grid, r] += inc
                e0[r].view(CHANNELS, BLOCKS, RANKS)[ch, :grid, t] += inc
        ck.true(f"{tag} signal pads", torch.equal(self.pads, p0), f"rank {r}: pad entries moved other than +{inc} "
                f"at [{ch}][b < {grid}][{r}] of the other members {list(self.members)}")
        ck.true(f"{tag} epochs", torch.equal(self.epochs, e0), f"rank {r}: epoch entries moved other than +{inc} "
                f"at the other members {list(self.members)}")
        if uncredited is None:
            box = list(self.box[:4])
            assert box == [0, 0, 0, 0], f"{tag}: rank {r} set the mailbox {box}"


def _groups(W, G):
    return [list(range(k * G, (k + 1) * G)) for k in range(W // G)]


def _symm():
    from distributed_torch_horovod_gcp_b200.runtime import symm as S
    return S


RS_GRIDS = {2: (7, 2 * 7 * THREADS - 1), 4: (1, 2 * THREADS + 1), 8: (128, 333)}   # G -> (grid, chunk vectors)


@gpu
@pytest.mark.parametrize("skind", ["inv", "inv3"])
@pytest.mark.parametrize("dtype", [F32, BF16, F16], ids=["f32", "bf16", "f16"])
@pytest.mark.parametrize("W,G", WG, ids=[f"w{W}-g{G}" for W, G in WG])
def test_group_reduce_scatter(W, G, dtype, skind):
    """``skind``: scale 1/G (what the runtime passes; exact in fp32 for these G), or 1/(3G), which fp32 does not
    hold exactly, so the bound's |sigma - scale| term is exercised."""
    S = _symm()
    grid, cvec = RS_GRIDS[G]
    chunk = cvec * VN[dtype]
    gen = torch.Generator().manual_seed(zlib.crc32(f"rs{W}{G}{dtype}{skind}".encode()))
    gs = make_grads(W, G * chunk, dtype, gen)                         # world rank w's staged input
    emu, ck = GroupEmu(W, seed=W * 10 + G), Checker()
    src, dst = [_buf(G * chunk, dtype, g) for g in gs], [_buf(chunk, dtype) for _ in range(W)]
    scale = 1.0 / G if skind == "inv" else 1.0 / (3 * G)
    for members in _groups(W, G):
        emu.members = members

        def fn(r, ctx, members=members):
            a = S.group_coll_args(members, members.index(r), [src[w].data_ptr() for w in members],
                                  [dst[w].data_ptr() for w in members], chunk, scale)
            return emu.lib.b200dp_comm_group_collective(ctypes.byref(ctx), ctypes.byref(a), S.COLL_REDUCE_SCATTER,
                                                        DT_CODE[dtype], grid, THREADS, _stream())
        fin, owner = emu.isolated(ck, "group reduce-scatter", {"src": src, "dst": dst}, fn, CH_USER, grid)
        for w in range(W):
            ck.true("group reduce-scatter src untouched", bool((owner["src"][w] == -1).all()), f"rank {w}")
            if w not in members:
                ck.true("group reduce-scatter non-member untouched", bool((owner["dst"][w] == -1).all()),
                        f"rank {w}, group {members}")
                continue
            g = members.index(w)
            check_sum(ck, f"group reduce-scatter {str(dtype)[6:]}", fin["dst"][w][:chunk],
                      [gs[m][g * chunk:(g + 1) * chunk] for m in members], fp32(scale), scale, dtype)
            ck.true("group reduce-scatter write set", owned_by(owner["dst"][w], torch.full((chunk,), w,
                                                                                            device="cuda")),
                    f"rank {w}")
    ck.close()


AG_GRIDS = {2: (1, 1), 4: (7, 7 * THREADS + 1), 8: (128, 128 * THREADS - 1)}       # G -> (grid, vectors)


@gpu
@pytest.mark.parametrize("W,G", WG, ids=[f"w{W}-g{G}" for W, G in WG])
def test_group_allgather(W, G):
    S = _symm()
    grid, nvec = AG_GRIDS[G]
    emu, ck = GroupEmu(W, seed=W * 10 + G), Checker()
    i32 = torch.int32
    src = [_buf(nvec * 4, i32, pattern(w, 0, nvec)) for w in range(W)]
    dst = [_buf(G * nvec * 4, i32) for _ in range(W)]
    for members in _groups(W, G):
        emu.members = members

        def fn(r, ctx, members=members):
            a = S.group_coll_args(members, members.index(r), [src[w].data_ptr() for w in members],
                                  [dst[w].data_ptr() for w in members], nvec)
            return emu.lib.b200dp_comm_group_collective(ctypes.byref(ctx), ctypes.byref(a), S.COLL_ALLGATHER, 0,
                                                        grid, THREADS, _stream())
        before = [t.clone() for t in dst]
        fin, owner = emu.isolated(ck, "group all-gather", {"src": src, "dst": dst}, fn, CH_USER, grid)
        want = torch.cat([pattern(w, 0, nvec) for w in members])
        slots = torch.tensor(members, device="cuda").repeat_interleave(nvec * 4)
        for w in range(W):
            ck.true("group all-gather src untouched", bool((owner["src"][w] == -1).all()), f"rank {w}")
            if w not in members:
                ck.same_bits("group all-gather non-member untouched", fin["dst"][w], before[w])
                continue
            ck.same_bits("group all-gather slots", fin["dst"][w][:G * nvec * 4], want)
            ck.true("group all-gather write set", owned_by(owner["dst"][w], slots), f"rank {w}")
    ck.close()


@gpu
@pytest.mark.parametrize("kernel", ["reduce-scatter", "allgather"])
def test_group_watchdog_exit_writes_nothing(kernel):
    """Group {2, 3, 5} of a world of 6 (members need not be contiguous for the kernels), rank 3 launched with the
    mailbox already set and member 5 uncredited: the opening barrier gives up after its spin limit and nothing is
    written."""
    S = _symm()
    W, grid, dtype, members, r = 6, 7, BF16, [2, 3, 5], 3
    G = len(members)
    chunk = (2 * 7 * THREADS + 5) * 8
    gen = torch.Generator().manual_seed(9)
    gs = make_grads(W, G * chunk, dtype, gen)
    emu, ck = GroupEmu(W, seed=3), Checker()
    emu.members = members
    src = [_buf(G * chunk, dtype, g) for g in gs]
    dst = [_buf(G * chunk, dtype) for _ in range(W)]

    def fn(ctx):
        mode = S.COLL_REDUCE_SCATTER if kernel == "reduce-scatter" else S.COLL_ALLGATHER
        a = S.group_coll_args(members, members.index(r), [src[w].data_ptr() for w in members],
                              [dst[w].data_ptr() for w in members], chunk if mode == 0 else chunk // 8)
        return emu.lib.b200dp_comm_group_collective(ctypes.byref(ctx), ctypes.byref(a), mode, DT_CODE[dtype], grid,
                                                    THREADS, _stream())
    before = [t.clone() for t in src + dst]
    box = emu.box
    box[0] = 1
    try:
        emu.launch(ck, f"group watchdog {kernel}", r, fn, CH_USER, grid, uncredited=5)
    finally:
        for i in range(4):
            box[i] = 0
    for t, t0 in zip(src + dst, before):
        ck.same_bits(f"group watchdog {kernel} writes nothing", t, t0)
    ck.close()
