"""Static gradient-bucket planner.

Replaces Horovod's runtime tensor fusion (fusion-buffer manager + response cache +
coordinator negotiation; SURVEY.md §2.2 N2/N4/N5).  Because every data-parallel rank
runs the same model, the plan is computed ONCE, deterministically, from the parameter
list; its hash is cross-checked over the control plane at construction, which replaces
Horovod's per-step negotiation check.  Gradients are *views* into the flat bucket, so the
``BatchedD2DMemcpy`` pack/unpack kernels of Horovod (N6) do not exist here.

Layout rules (they matter to the sm_90a kernels in csrc/comm_kernels.cu):
  * a bucket never mixes dtypes, devices or optimizer param-groups (one hyper-parameter
    block per bucket);
  * every tensor starts on a 16-byte boundary inside the bucket (vectorised 128-bit
    access even for the reference model's 4-byte and 256-byte gradients — SURVEY §2.6);
  * bucket sizes are padded to ``ALIGN_ELEMS`` so that W-way slicing (two-shot / NVLS)
    yields 16-byte-aligned slices for every world size up to 8;
  * parameters are placed in *reverse* registration order, which approximates backward
    readiness order, so the first bucket to fill is the one whose gradients arrive first.
"""
from __future__ import annotations

import hashlib
import os
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Sequence, Tuple

import torch

ALIGN_BYTES = 16
SLICE_ALIGN_BYTES = 16 * 8 * 32  # each of up to 8 rank-slices stays 512B-aligned


def default_bucket_bytes() -> int:
    """Bucket capacity.  ``HOROVOD_FUSION_THRESHOLD`` (bytes) is honoured for parity with
    Horovod's knob; default 16 MiB: on NVSwitch every peer is reachable at full bandwidth,
    so buckets are sized for launch latency / overlap granularity, not for link count."""
    v = os.environ.get("B200DP_BUCKET_BYTES") or os.environ.get("HOROVOD_FUSION_THRESHOLD")
    if v:
        try:
            return max(int(v), 1024)
        except ValueError:
            pass
    return 16 << 20


@dataclass
class Slot:
    name: str
    param: torch.nn.Parameter
    offset: int          # element offset inside the bucket
    numel: int
    group_index: int


@dataclass
class Bucket:
    index: int
    dtype: torch.dtype
    device: torch.device
    group_index: int
    slots: List[Slot] = field(default_factory=list)
    numel: int = 0        # padded element count
    flat_offset: int = 0  # element offset inside the per-(dtype,device) flat arena

    @property
    def nbytes(self) -> int:
        return self.numel * torch.empty((), dtype=self.dtype).element_size()


def _pad(n_elems: int, esize: int, align_bytes: int) -> int:
    a = max(align_bytes // esize, 1)
    return (n_elems + a - 1) // a * a


def plan_buckets(named_params: Sequence[Tuple[str, torch.nn.Parameter]],
                 group_of: Dict[int, int],
                 bucket_bytes: Optional[int] = None,
                 explicit_groups: Optional[List[List[torch.nn.Parameter]]] = None,
                 num_groups: int = 0,
                 grad_dtype: Optional[torch.dtype] = None) -> List[Bucket]:
    """Build the bucket list.

    named_params : parameters that require grad, in registration order.
    group_of     : id(param) -> optimizer param-group index.
    explicit_groups / num_groups : Horovod's ``groups=`` / ``num_groups=`` arguments.
    grad_dtype   : wire/storage dtype of gradients (None = same as the parameter).
    """
    bucket_bytes = bucket_bytes or default_bucket_bytes()
    order = list(reversed(list(named_params)))
    buckets: List[Bucket] = []

    def new_bucket(dtype, device, gidx) -> Bucket:
        b = Bucket(index=len(buckets), dtype=dtype, device=device, group_index=gidx)
        buckets.append(b)
        return b

    def add(b: Bucket, name: str, p: torch.nn.Parameter):
        esize = torch.empty((), dtype=b.dtype).element_size()
        off = _pad(b.numel, esize, ALIGN_BYTES)
        b.slots.append(Slot(name, p, off, p.numel(), b.group_index))
        b.numel = off + p.numel()

    if explicit_groups:
        name_of = {id(p): n for n, p in named_params}
        seen = set()
        for grp in explicit_groups:
            cur: Dict[Tuple, Bucket] = {}
            for p in grp:
                if id(p) not in name_of:
                    continue
                seen.add(id(p))
                dt = grad_dtype or p.dtype
                key = (dt, p.device, group_of.get(id(p), 0))
                if key not in cur:
                    cur[key] = new_bucket(*key)
                add(cur[key], name_of[id(p)], p)
        order = [(n, p) for n, p in order if id(p) not in seen]

    if num_groups and num_groups > 0 and order:
        total = sum(p.numel() * p.element_size() for _, p in order)
        bucket_bytes = max((total + num_groups - 1) // num_groups, 1)

    open_b: Dict[Tuple, Bucket] = {}
    for name, p in order:
        dt = grad_dtype or p.dtype
        key = (dt, p.device, group_of.get(id(p), 0))
        esize = torch.empty((), dtype=dt).element_size()
        b = open_b.get(key)
        if b is None or (b.numel > 0 and (b.numel + p.numel()) * esize > bucket_bytes):
            b = new_bucket(*key)
            open_b[key] = b
        add(b, name, p)

    buckets = [b for b in buckets if b.slots]
    for i, b in enumerate(buckets):
        b.index = i
        esize = torch.empty((), dtype=b.dtype).element_size()
        b.numel = _pad(b.numel, esize, SLICE_ALIGN_BYTES)
    # flat arena offsets per (dtype, device)
    arena: Dict[Tuple, int] = {}
    for b in buckets:
        k = (b.dtype, b.device)
        b.flat_offset = arena.get(k, 0)
        arena[k] = b.flat_offset + b.numel
    return buckets


def arena_sizes(buckets: Sequence[Bucket]) -> Dict[Tuple[torch.dtype, torch.device], int]:
    out: Dict[Tuple, int] = {}
    for b in buckets:
        k = (b.dtype, b.device)
        out[k] = max(out.get(k, 0), b.flat_offset + b.numel)
    return out


def plan_hash(buckets: Sequence[Bucket]) -> str:
    """Deterministic digest of the plan; compared across ranks at construction so a
    divergent model/plan fails fast instead of hanging inside a kernel (SURVEY §5.2)."""
    h = hashlib.sha256()
    for b in buckets:
        h.update(f"B{b.index}|{b.dtype}|{b.group_index}|{b.numel}|{b.flat_offset};".encode())
        for s in b.slots:
            h.update(f"{s.name}:{s.offset}:{s.numel}:{tuple(s.param.shape)};".encode())
    return h.hexdigest()
