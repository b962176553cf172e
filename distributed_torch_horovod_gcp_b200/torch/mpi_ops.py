"""Collective operations with Horovod's call shapes (``allreduce[_async][_]``, ``broadcast``,
``allgather``, ``alltoall``, ``reducescatter``, ``synchronize``/``poll``, ``barrier``, ``join``).

Replaces Horovod's torch binding + tensor queue + handle manager (SURVEY.md §2.2 N3, N7,
N8, N10; used by the reference through app/torch_train.py:259,266).

Data plane selection per tensor:
  * CPU tensor            -> Gloo (``torch.distributed``), the CPU plumbing configuration.
  * CUDA tensor           -> symmetric-memory sm_90a kernels (one-shot / two-shot / NVLS
                             allreduce, multicast broadcast, reduce-scatter, all-gather,
                             equal-split all-to-all) from ``runtime.symm``; ragged all-gather /
                             all-to-all shapes keep the torch.distributed path.
  * CUDA tensor, no symm  -> NCCL fallback (warned once at runtime creation).

Handles are small integers, as in Horovod.  For CUDA work a handle wraps a CUDA event;
``synchronize`` makes the *current stream* wait on it (stream-ordered, no host stall)
and additionally blocks the host only when ``HOROVOD_SYNC_HOST=1``.
"""
from __future__ import annotations

import itertools
import os
import threading
from typing import Dict, List, Optional, Sequence, Tuple

import torch
import torch.distributed as dist

from .. import _state
from .compression import Compression


class _ReduceOp:
    def __init__(self, name: str, value: int):
        self.name, self.value = name, value

    def __repr__(self):
        return f"hvd.{self.name}"


Average = _ReduceOp("Average", 0)
Sum = _ReduceOp("Sum", 1)
Adasum = _ReduceOp("Adasum", 2)
Min = _ReduceOp("Min", 3)
Max = _ReduceOp("Max", 4)
Product = _ReduceOp("Product", 5)

_DIST_OP = {
    0: dist.ReduceOp.SUM, 1: dist.ReduceOp.SUM, 3: dist.ReduceOp.MIN,
    4: dist.ReduceOp.MAX, 5: dist.ReduceOp.PRODUCT,
}


class HorovodInternalError(RuntimeError):
    """Raised when a collective fails (peer died / watchdog timeout); elastic mode catches it."""


# ----------------------------------------------------------------------------- handles
class _Handle:
    __slots__ = ("work", "event", "stream", "output", "post", "name", "done")

    def __init__(self, output, work=None, event=None, stream=None, post=None, name=None):
        self.output, self.work, self.event, self.stream = output, work, event, stream
        self.post, self.name, self.done = post, name, False


class _HandleManager:
    """Thread-safe integer-handle table (Horovod's HandleManager equivalent)."""

    def __init__(self):
        self._lock = threading.Lock()
        self._next = itertools.count(1)
        self._table: Dict[int, _Handle] = {}
        self._names: Dict[str, int] = {}

    def add(self, h: _Handle) -> int:
        with self._lock:
            if h.name is not None:
                if h.name in self._names:
                    raise ValueError(
                        f"Duplicate tensor name '{h.name}': a collective with this name is "
                        "already in flight; names must be unique among outstanding operations.")
                i = next(self._next)
                self._names[h.name] = i
            else:
                i = next(self._next)
            self._table[i] = h
            return i

    def get(self, i: int) -> _Handle:
        with self._lock:
            if i not in self._table:
                raise ValueError(f"Handle {i} was not created or has been cleared.")
            return self._table[i]

    def pop(self, i: int) -> _Handle:
        with self._lock:
            if i not in self._table:
                raise ValueError(f"Handle {i} was not created or has been cleared.")
            h = self._table.pop(i)
            if h.name is not None:
                self._names.pop(h.name, None)
            return h

    def outstanding(self) -> int:
        with self._lock:
            return len(self._table)


_handles = _HandleManager()


def _finish(h: _Handle):
    if h.done:
        return h.output
    try:
        if h.work is not None:
            h.work.wait()
        if h.event is not None:
            torch.cuda.current_stream(h.output.device if isinstance(h.output, torch.Tensor)
                                      else None).wait_event(h.event)
            if os.environ.get("HOROVOD_SYNC_HOST", "0") == "1":
                h.event.synchronize()
            symm = _state.runtime().symm
            if symm is not None:
                symm.check_errors()     # a bounded spin-wait expired in an earlier kernel (host-mapped mailbox)
    except RuntimeError as e:  # surfaced collective failure
        raise HorovodInternalError(str(e)) from e
    if h.post is not None:
        h.output = h.post(h.output)
        h.post = None
    h.done = True
    return h.output


def poll(handle: int) -> bool:
    """True when the operation behind ``handle`` has completed (non-blocking)."""
    h = _handles.get(handle)
    if h.done:
        return True
    if h.work is not None and not h.work.is_completed():
        return False
    if h.event is not None and not h.event.query():
        return False
    return True


def synchronize(handle: int):
    """Wait for an async op and return its output tensor (Horovod ``hvd.synchronize``)."""
    h = _handles.pop(handle)
    return _finish(h)


# ----------------------------------------------------------------------------- helpers
def _rt():
    return _state._require_init()


def _group_for(t: torch.Tensor, process_set=None):
    rt = _rt()
    if process_set is not None and getattr(process_set, "group", None) is not None:
        return process_set.group
    if t.is_cuda:
        return dist.group.WORLD
    return rt.cpu_group if rt.cpu_group is not None else dist.group.WORLD


def _ps_size(process_set) -> int:
    if process_set is not None and getattr(process_set, "ranks", None):
        return len(process_set.ranks)
    return _rt().size


def _check_op(op):
    if op is Adasum or getattr(op, "value", None) == 2:
        raise NotImplementedError(
            "op=Adasum is not implemented in the H100 runtime (Average/Sum/Min/Max/Product are).")


def _timeline(name: str, phase: str, **kw):
    tl = _state.runtime().timeline
    if tl is not None:
        tl.mark(name or "unnamed", phase, **kw)
    from ..utils import nvtx
    if nvtx.enabled():
        nvtx.mark(f"{phase} {name or 'unnamed'}")


# ----------------------------------------------------------------------------- allreduce
def _allreduce_impl(tensor: torch.Tensor, output: torch.Tensor, op, prescale: float,
                    postscale: float, name: Optional[str], process_set, async_: bool,
                    lane: int = 0) -> _Handle:
    _check_op(op)
    rt = _rt()
    n = _ps_size(process_set)
    if op is Average:
        postscale = postscale / n
    if output.data_ptr() != tensor.data_ptr():
        output.copy_(tensor)
    if n == 1:
        if prescale * postscale != 1.0:
            output.mul_(prescale * postscale)
        return _Handle(output, name=name)
    _timeline(name, "ALLREDUCE_BEGIN", bytes=output.numel() * output.element_size())
    if output.is_cuda and process_set is None:
        symm = _state.get_symm()
        if symm is not None and op.value in (0, 1) and symm.supports(output.dtype):
            ev = symm.allreduce_(output, prescale=prescale, postscale=postscale, lane=lane)
            return _Handle(output, event=ev, name=name)
    if prescale != 1.0:
        output.mul_(prescale)
    work = dist.all_reduce(output, op=_DIST_OP[op.value], group=_group_for(output, process_set),
                           async_op=True)
    post = None
    if postscale != 1.0:
        if output.is_floating_point() or output.is_complex():
            post = lambda o: o.mul_(postscale)
        else:
            post = lambda o: o.copy_((o.to(torch.float64) * postscale).to(o.dtype))
    return _Handle(output, work=work, post=post, name=name)


def allreduce_async(tensor, average=None, name=None, op=None, prescale_factor=1.0,
                    postscale_factor=1.0, process_set=None) -> int:
    op = _resolve_op(average, op)
    out = torch.empty_like(tensor)
    return _handles.add(_allreduce_impl(tensor, out, op, prescale_factor, postscale_factor,
                                        name, process_set, True))


def allreduce_async_(tensor, average=None, name=None, op=None, prescale_factor=1.0,
                     postscale_factor=1.0, process_set=None, _lane: int = 0) -> int:
    """``_lane`` (internal): 1 = DistributedOptimizer's side-stream bucket path, which gets its own
    staging buffer and barrier channel so it can overlap user collectives on the main stream."""
    op = _resolve_op(average, op)
    return _handles.add(_allreduce_impl(tensor, tensor, op, prescale_factor, postscale_factor,
                                        name, process_set, True, lane=_lane))


def _resolve_op(average, op):
    if average is not None and op is not None:
        raise ValueError("The op parameter supersedes average; provide only one of them.")
    if op is None:
        op = Average if (average is None or average) else Sum
    return op


class _AllreduceFn(torch.autograd.Function):
    """Differentiable allreduce: the gradient of an allreduce is an allreduce (Horovod parity)."""

    @staticmethod
    def forward(ctx, tensor, average, name, op, prescale, postscale, process_set):
        ctx.args = (average, op, prescale, postscale, process_set)
        return synchronize(allreduce_async(tensor, average, name, op, prescale, postscale,
                                           process_set))

    @staticmethod
    def backward(ctx, grad):
        average, op, prescale, postscale, ps = ctx.args
        g = synchronize(allreduce_async(grad.contiguous(), average, None, op, prescale,
                                        postscale, ps))
        return g, None, None, None, None, None, None


def allreduce(tensor, average=None, name=None, compression=Compression.none, op=None,
              prescale_factor=1.0, postscale_factor=1.0, process_set=None):
    """Out-of-place allreduce; averaged by default.  The [DRIVER] north star names this as
    the fourth public op (BASELINE.json; SURVEY.md §2.3)."""
    t, ctx = compression.compress(tensor)
    if t.requires_grad:
        out = _AllreduceFn.apply(t, average, name, op, prescale_factor, postscale_factor,
                                 process_set)
    else:
        out = synchronize(allreduce_async(t, average, name, op, prescale_factor,
                                          postscale_factor, process_set))
    return compression.decompress(out, ctx)


def allreduce_(tensor, average=None, name=None, op=None, prescale_factor=1.0,
               postscale_factor=1.0, process_set=None):
    return synchronize(allreduce_async_(tensor, average, name, op, prescale_factor,
                                        postscale_factor, process_set))


def grouped_allreduce_async(tensors: Sequence[torch.Tensor], average=None, name=None, op=None,
                            prescale_factor=1.0, postscale_factor=1.0, process_set=None) -> int:
    outs = [torch.empty_like(t) for t in tensors]
    for o, t in zip(outs, tensors):
        o.copy_(t)
    return grouped_allreduce_async_(outs, average, name, op, prescale_factor, postscale_factor,
                                    process_set)


def grouped_allreduce_async_(tensors: Sequence[torch.Tensor], average=None, name=None, op=None,
                             prescale_factor=1.0, postscale_factor=1.0, process_set=None) -> int:
    """Fused allreduce of a tensor group: same-dtype tensors are packed into ONE flat
    buffer and reduced with ONE collective (explicit tensor fusion — SURVEY.md §2.2 N5)."""
    op = _resolve_op(average, op)
    tensors = list(tensors)
    if not tensors:
        return _handles.add(_Handle([], name=name))
    by_key: Dict[Tuple, List[int]] = {}
    for i, t in enumerate(tensors):
        by_key.setdefault((t.dtype, t.device), []).append(i)
    subs: List[Tuple[_Handle, List[int], torch.Tensor]] = []
    for (dtype, device), idxs in by_key.items():
        flat = torch.cat([tensors[i].reshape(-1) for i in idxs])
        h = _allreduce_impl(flat, flat, op, prescale_factor, postscale_factor, None,
                            process_set, True)
        subs.append((h, idxs, flat))

    def post(_):
        for h, idxs, flat in subs:
            _finish(h)
            off = 0
            for i in idxs:
                n = tensors[i].numel()
                tensors[i].copy_(flat[off:off + n].view_as(tensors[i]))
                off += n
        return tensors

    return _handles.add(_Handle(tensors, post=post, name=name))


def grouped_allreduce(tensors, average=None, name=None, compression=Compression.none, op=None,
                      prescale_factor=1.0, postscale_factor=1.0, process_set=None):
    comp, ctxs = zip(*[compression.compress(t) for t in tensors]) if tensors else ((), ())
    outs = synchronize(grouped_allreduce_async(list(comp), average, name, op, prescale_factor,
                                               postscale_factor, process_set))
    return [compression.decompress(o, c) for o, c in zip(outs, ctxs)]


def grouped_allreduce_(tensors, average=None, name=None, op=None, prescale_factor=1.0,
                       postscale_factor=1.0, process_set=None):
    return synchronize(grouped_allreduce_async_(tensors, average, name, op, prescale_factor,
                                                postscale_factor, process_set))


# ----------------------------------------------------------------------------- broadcast
def _broadcast_impl(tensor: torch.Tensor, output: torch.Tensor, root_rank: int,
                    name: Optional[str], process_set) -> _Handle:
    rt = _rt()
    n = _ps_size(process_set)
    if not (0 <= root_rank < rt.size):
        raise ValueError(f"root_rank {root_rank} out of range for size {rt.size}")
    if output.data_ptr() != tensor.data_ptr():
        output.copy_(tensor)
    if n == 1:
        return _Handle(output, name=name)
    _timeline(name, "BROADCAST_BEGIN", bytes=output.numel() * output.element_size())
    if output.is_cuda and process_set is None and output.is_contiguous():
        symm = _state.get_symm()
        if symm is not None:
            ev = symm.broadcast_(output, root_rank)
            return _Handle(output, event=ev, name=name)
    if not output.is_contiguous():
        tmp = output.contiguous()
        work = dist.broadcast(tmp, src=root_rank, group=_group_for(tmp, process_set),
                              async_op=True)
        return _Handle(output, work=work, post=lambda o: o.copy_(tmp), name=name)
    work = dist.broadcast(output, src=root_rank, group=_group_for(output, process_set),
                          async_op=True)
    return _Handle(output, work=work, name=name)


def broadcast_async(tensor, root_rank, name=None, process_set=None) -> int:
    out = torch.empty_like(tensor)
    return _handles.add(_broadcast_impl(tensor, out, root_rank, name, process_set))


def broadcast_async_(tensor, root_rank, name=None, process_set=None) -> int:
    return _handles.add(_broadcast_impl(tensor, tensor, root_rank, name, process_set))


def broadcast(tensor, root_rank, name=None, process_set=None):
    return synchronize(broadcast_async(tensor, root_rank, name, process_set))


def broadcast_(tensor, root_rank, name=None, process_set=None):
    return synchronize(broadcast_async_(tensor, root_rank, name, process_set))


# ----------------------------------------------------------------------------- allgather
def allgather_async(tensor, name=None, process_set=None) -> int:
    """Concatenate along dim 0; first dimensions may differ across ranks (Horovod semantics)."""
    rt = _rt()
    n = _ps_size(process_set)
    if tensor.dim() == 0:
        tensor = tensor.reshape(1)
    if n == 1:
        return _handles.add(_Handle(tensor.clone(), name=name))
    group = _group_for(tensor, process_set)
    sizes = [None] * n
    dist.all_gather_object(sizes, int(tensor.shape[0]),
                           group=group if not tensor.is_cuda else
                           (process_set.group if process_set is not None and process_set.group
                            else rt.cpu_group))
    mx = max(sizes)
    symm = _state.get_symm() if (tensor.is_cuda and process_set is None) else None
    row_bytes = (tensor.numel() // max(tensor.shape[0], 1)) * tensor.element_size() if tensor.shape[0] else 0
    if symm is not None and min(sizes) == mx and mx > 0 and (mx * row_bytes) % 16 == 0:
        # equal shards: every rank pushes its shard into slot `rank` of all peers over NVLink (sm_90a kernel)
        src = tensor.contiguous()
        out = torch.empty((n * mx,) + tuple(tensor.shape[1:]), dtype=tensor.dtype, device=tensor.device)
        ev = symm.allgather(src, out)
        return _handles.add(_Handle(out, event=ev, name=name))
    pad = tensor
    if tensor.shape[0] != mx:
        pad = torch.zeros((mx,) + tuple(tensor.shape[1:]), dtype=tensor.dtype,
                          device=tensor.device)
        pad[: tensor.shape[0]] = tensor
    outs = [torch.empty_like(pad) for _ in range(n)]
    work = dist.all_gather(outs, pad.contiguous(), group=group, async_op=True)

    def post(_):
        return torch.cat([o[:s] for o, s in zip(outs, sizes)], dim=0)

    return _handles.add(_Handle(None, work=work, post=post, name=name))


def allgather(tensor, name=None, process_set=None):
    return synchronize(allgather_async(tensor, name, process_set))


def grouped_allgather(tensors, name=None, process_set=None):
    return [allgather(t, None, process_set) for t in tensors]


# ----------------------------------------------------------------------------- alltoall
def alltoall_async(tensor, splits=None, name=None, process_set=None) -> int:
    rt = _rt()
    n = _ps_size(process_set)
    if n == 1:
        out = tensor.clone()
        rs = torch.tensor([tensor.shape[0]], dtype=torch.int32)
        return _handles.add(_Handle((out, rs) if splits is not None else out, name=name))
    if splits is None:
        if tensor.shape[0] % n != 0:
            raise ValueError("alltoall without splits needs dim 0 divisible by the world size")
        send = [tensor.shape[0] // n] * n
    else:
        send = [int(s) for s in (splits.tolist() if isinstance(splits, torch.Tensor) else splits)]
        if len(send) != n or sum(send) != tensor.shape[0]:
            raise ValueError("splits must have one entry per rank and sum to tensor.shape[0]")
    if splits is None and tensor.is_cuda and process_set is None:
        symm = _state.get_symm()
        per = tensor.numel() // n * tensor.element_size()
        if symm is not None and per > 0 and per % 16 == 0:
            src = tensor.contiguous()
            out = torch.empty_like(src)
            ev = symm.alltoall(src, out)
            return _handles.add(_Handle(out, event=ev, name=name))
    ctl = process_set.group if process_set is not None and process_set.group else rt.cpu_group
    all_send = [None] * n
    dist.all_gather_object(all_send, send, group=ctl)
    my = dist.get_rank(ctl) if ctl is not None else rt.rank
    recv = [all_send[r][my] for r in range(n)]
    ins = list(torch.split(tensor.contiguous(), send, dim=0))
    outs = [torch.empty((r,) + tuple(tensor.shape[1:]), dtype=tensor.dtype, device=tensor.device)
            for r in recv]
    group = _group_for(tensor, process_set)
    if tensor.is_cuda:
        work = dist.all_to_all(outs, ins, group=group, async_op=True)
    else:
        # Gloo has no all_to_all for lists on every build: emulate with isend/irecv.
        reqs = []
        for r in range(n):
            if r == my:
                outs[r].copy_(ins[r])
            else:
                gr = dist.get_global_rank(group, r) if group is not dist.group.WORLD else r
                reqs.append(dist.isend(ins[r], gr, group=group))
                reqs.append(dist.irecv(outs[r], gr, group=group))

        class _Multi:
            def wait(self_inner):
                for q in reqs:
                    q.wait()

            def is_completed(self_inner):
                return all(q.is_completed() for q in reqs)
        work = _Multi()

    def post(_):
        out = torch.cat(outs, dim=0)
        if splits is not None:
            return out, torch.tensor(recv, dtype=torch.int32)
        return out

    return _handles.add(_Handle(None, work=work, post=post, name=name))


def alltoall(tensor, splits=None, name=None, process_set=None):
    return synchronize(alltoall_async(tensor, splits, name, process_set))


# ----------------------------------------------------------------------------- reducescatter
def reducescatter_async(tensor, name=None, op=None, process_set=None, prescale_factor=1.0,
                        postscale_factor=1.0) -> int:
    op = Average if op is None else op
    _check_op(op)
    n = _ps_size(process_set)
    if n == 1:
        return _handles.add(_Handle(tensor.clone() * (prescale_factor * postscale_factor),
                                    name=name))
    rows = tensor.shape[0]
    base, rem = divmod(rows, n)
    counts = [base + (1 if r < rem else 0) for r in range(n)]
    if tensor.is_cuda and process_set is None and rem == 0 and op.value in (0, 1):
        symm = _state.get_symm()
        per = tensor.numel() // n
        if symm is not None and symm.supports(tensor.dtype) and per > 0 and \
                (per * tensor.element_size()) % 16 == 0:
            # rank r reads only chunk r of every peer (or the NVSwitch sums it): S*(N-1)/N bytes, not 2S
            src = tensor.contiguous()
            out = torch.empty((base,) + tuple(tensor.shape[1:]), dtype=tensor.dtype, device=tensor.device)
            scale = prescale_factor * postscale_factor / (n if op is Average else 1)
            ev = symm.reducescatter(src, out, scale)
            return _handles.add(_Handle(out, event=ev, name=name))
    full = tensor.clone()
    if prescale_factor != 1.0:
        full.mul_(prescale_factor)
    group = _group_for(tensor, process_set)
    work = dist.all_reduce(full, op=_DIST_OP[op.value], group=group, async_op=True)
    my = dist.get_rank(group)

    def post(_):
        start = sum(counts[:my])
        out = full[start:start + counts[my]].clone()
        scale = postscale_factor / (n if op is Average else 1)
        if scale != 1.0:
            out.mul_(scale)
        return out

    return _handles.add(_Handle(None, work=work, post=post, name=name))


def reducescatter(tensor, name=None, compression=Compression.none, op=None, process_set=None,
                  prescale_factor=1.0, postscale_factor=1.0):
    t, ctx = compression.compress(tensor)
    out = synchronize(reducescatter_async(t, name, op, process_set, prescale_factor,
                                          postscale_factor))
    return compression.decompress(out, ctx)


def grouped_reducescatter(tensors, name=None, compression=Compression.none, op=None,
                          process_set=None, prescale_factor=1.0, postscale_factor=1.0):
    return [reducescatter(t, None, compression, op, process_set, prescale_factor,
                          postscale_factor) for t in tensors]


# ----------------------------------------------------------------------------- barrier / join
def barrier(process_set=None) -> None:
    rt = _rt()
    if _ps_size(process_set) == 1:
        return
    g = process_set.group if process_set is not None and process_set.group else rt.cpu_group
    dist.barrier(group=g)


def join(device: int = -1) -> int:
    """Block until every rank has called ``join``; returns the last rank to arrive.
    (Uneven-data support: ranks that ran out of batches call join while others finish.)"""
    rt = _rt()
    if rt.size == 1:
        return 0
    import time
    stamp = torch.tensor([time.time()], dtype=torch.float64)
    stamps = [torch.zeros(1, dtype=torch.float64) for _ in range(rt.size)]
    dist.all_gather(stamps, stamp, group=rt.cpu_group)
    return int(max(range(rt.size), key=lambda r: stamps[r].item()))
