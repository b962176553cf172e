"""``broadcast_parameters`` / ``broadcast_optimizer_state`` / ``broadcast_object`` /
``allgather_object`` (Horovod ``horovod/torch/functions.py`` call shapes).

``broadcast_parameters`` is the startup collective of the reference
(app/torch_train.py:266; semantics SURVEY.md §2.3 A7).  H100-first difference: instead of
one ``ncclBcast`` per tensor, all CUDA tensors of a dtype are packed into ONE flat
symmetric buffer and broadcast by ONE multicast-store kernel (K4, csrc/comm_kernels.cu);
the 10 tensors / 1.48 MB of the reference model therefore cost a single launch.
"""
from __future__ import annotations

import collections
import io
import pickle
from typing import Dict, List, Tuple

import torch
import torch.distributed as dist

from .. import _state
from . import mpi_ops


def _named_tensors(params) -> List[Tuple[str, torch.Tensor]]:
    if isinstance(params, dict):
        items = sorted(params.items())
    elif isinstance(params, list) or hasattr(params, "__iter__"):
        items = list(params)
        if items and not (isinstance(items[0], tuple) and len(items[0]) == 2):
            raise ValueError("invalid params of type: %s" % type(params))
        items = [(n, p) for n, p in items]
    else:
        raise ValueError("invalid params of type: %s" % type(params))
    out = []
    for name, p in items:
        if p is None:
            continue
        if not isinstance(p, torch.Tensor):
            raise ValueError(f"invalid params: entry '{name}' is {type(p)}, expected a tensor")
        out.append((name, p))
    return out


def broadcast_parameters(params, root_rank: int, process_set=None) -> None:
    """Broadcast ``model.state_dict()`` / ``named_parameters()`` (parameters **and**
    buffers) from ``root_rank`` to all ranks, in place."""
    rt = _state._require_init()
    items = _named_tensors(params)
    if mpi_ops._ps_size(process_set) == 1 or not items:
        _refresh_engines()
        return
    # fused path: pack by (dtype, device) -> one broadcast each
    groups: Dict[Tuple, List[torch.Tensor]] = collections.OrderedDict()
    for name, t in items:
        tt = t.data if isinstance(t, torch.nn.Parameter) else t
        groups.setdefault((tt.dtype, tt.device), []).append(tt)
    handles = []
    for (dtype, device), ts in groups.items():
        if len(ts) == 1 and ts[0].is_contiguous():
            handles.append((mpi_ops.broadcast_async_(ts[0], root_rank, process_set=process_set),
                            None, None))
            continue
        flat = torch.cat([t.reshape(-1) for t in ts])
        handles.append((mpi_ops.broadcast_async_(flat, root_rank, process_set=process_set),
                        flat, ts))
    for h, flat, ts in handles:
        mpi_ops.synchronize(h)
        if flat is not None:
            off = 0
            for t in ts:
                n = t.numel()
                t.copy_(flat[off:off + n].view_as(t))
                off += n
    _refresh_engines()


def _refresh_engines() -> None:
    """Parameters may live in a fused engine's arena with a separate fp32 master copy: after
    they were (re)written from outside — this broadcast, or a checkpoint load followed by the
    customary ``broadcast_parameters`` — the masters are refreshed from the parameters."""
    from ..parallel.fused_engine import live_engines
    for eng in live_engines():
        eng.params_changed()


def broadcast_object(obj, root_rank: int = 0, name=None, process_set=None):
    """Pickle ``obj`` on root and broadcast it; returns the object on every rank."""
    rt = _state._require_init()
    if mpi_ops._ps_size(process_set) == 1:
        return obj
    if rt.rank == root_rank:
        buf = io.BytesIO()
        pickle.dump(obj, buf, protocol=pickle.HIGHEST_PROTOCOL)
        data = torch.frombuffer(bytearray(buf.getvalue()), dtype=torch.uint8)
        sz = torch.tensor([data.numel()], dtype=torch.int64)
    else:
        data, sz = None, torch.zeros(1, dtype=torch.int64)
    mpi_ops.broadcast_(sz, root_rank, process_set=process_set)
    if rt.rank != root_rank:
        data = torch.empty(int(sz.item()), dtype=torch.uint8)
    mpi_ops.broadcast_(data, root_rank, process_set=process_set)
    if rt.rank == root_rank:
        return obj
    return pickle.loads(data.numpy().tobytes())


def allgather_object(obj, name=None, process_set=None) -> list:
    rt = _state._require_init()
    n = mpi_ops._ps_size(process_set)
    if n == 1:
        return [obj]
    out = [None] * n
    g = process_set.group if process_set is not None and process_set.group else rt.cpu_group
    dist.all_gather_object(out, obj, group=g)
    return out


def broadcast_optimizer_state(optimizer, root_rank: int, model=None, process_set=None) -> None:
    """Broadcast optimizer hyper-parameters and per-parameter state from ``root_rank``.

    Not called by the reference (SURVEY.md §2.3 A7 notes its absence) but part of the
    checkpoint/resume convention "rank 0 loads, then broadcast" (SURVEY.md §5.4).
    """
    if isinstance(optimizer, torch.optim.LBFGS):
        raise ValueError("cannot broadcast torch.optim.LBFGS state")
    rt = _state._require_init()
    if mpi_ops._ps_size(process_set) == 1:
        return
    eng = getattr(optimizer, "fused_engine", None)
    if eng is not None:
        eng.export_state()
    state_dict = optimizer.state_dict()
    # structure (non-tensor part) goes through broadcast_object; tensors through broadcast_
    def strip(sd):
        tensors, skeleton = [], {"param_groups": sd["param_groups"], "state": {}}
        for pid, st in sorted(sd["state"].items(), key=lambda kv: str(kv[0])):
            skeleton["state"][pid] = {}
            for k, v in sorted(st.items()):
                if isinstance(v, torch.Tensor):
                    skeleton["state"][pid][k] = ("__tensor__", tuple(v.shape), str(v.dtype),
                                                 str(v.device))
                    tensors.append(((pid, k), v))
                else:
                    skeleton["state"][pid][k] = v
        return skeleton, tensors

    skeleton, tensors = strip(state_dict)
    skeleton = broadcast_object(skeleton, root_rank, process_set=process_set)
    if rt.rank != root_rank:
        # materialise missing state so load_state_dict has the right structure
        have = {key: t for key, t in tensors}
        tensors = []
        new_state = {}
        for pid, st in skeleton["state"].items():
            new_state[pid] = {}
            for k, v in st.items():
                if isinstance(v, tuple) and len(v) == 4 and v[0] == "__tensor__":
                    _, shape, dt, dev = v
                    dtype = getattr(torch, dt.replace("torch.", ""))
                    t = have.get((pid, k))
                    if t is None or tuple(t.shape) != tuple(shape) or t.dtype != dtype:
                        device = torch.device(dev) if not dev.startswith("cuda") else \
                            torch.device("cuda", torch.cuda.current_device())
                        t = torch.zeros(shape, dtype=dtype, device=device)
                    new_state[pid][k] = t
                    tensors.append(((pid, k), t))
                else:
                    new_state[pid][k] = v
        full = {"param_groups": skeleton["param_groups"], "state": new_state}
    else:
        full = None
    broadcast_parameters([(f"{pid}.{k}", t) for (pid, k), t in tensors], root_rank, process_set)
    if rt.rank != root_rank:
        optimizer.load_state_dict(full)
    if eng is not None:
        eng.import_state()
