"""Fused gradient-allreduce + optimizer engine (the north-star hot path).

One bucket == one launch of an sm_90a kernel from csrc/comm_kernels.cu that
  (1) reduces the bucket's gradients across all ranks by reading peer memory over NVLink
      (one-shot), or by slice with P2P pushes (two-shot), or in the NVSwitch (NVLS);
  (2) scales by 1/N, (3) runs the SGD-momentum / Adam / AdamW update on fp32 master
  weights + state, (4) writes the updated parameters in the model dtype (pushing them to
  every peer for the sliced algorithms) and (5) zeroes the consumed gradients —
on a high-priority side stream ordered after backward by an event, so ``optimizer.step()``
is a stream wait.  No NCCL, no separate scale kernel, no separate optimizer kernels, no
pack/unpack (SURVEY.md §2.2 N5-N7/N15, §2.6 S8-S10, §5.8; reference app/torch_train.py:
259,277,280-281).

Memory plan (per dtype arena, same element layout in every arena):
  G  gradients      symmetric   p.grad are views        (peers read / switch reduces)
  P  parameters     symmetric   p.data are views        (peers push updated slices)
  M  fp32 master    local       only when dtype != fp32
  S0 momentum | exp_avg,  S1 exp_avg_sq   local fp32    (sharded by slice for K2/K3)
"""
from __future__ import annotations

import weakref
from typing import Dict, List, Optional

import torch
import torch.distributed as dist

from .. import _state
from ..utils import nvtx
from .buckets import Bucket, arena_sizes

_ENGINES: "weakref.WeakSet[FusedEngine]" = weakref.WeakSet()


def live_engines():
    return list(_ENGINES)


def arena_view(flat: torch.Tensor, lo: int, param: torch.Tensor) -> torch.Tensor:
    """View of ``flat[lo: lo + numel]`` with the parameter's shape AND memory layout: a channels_last
    conv weight stays [Cout][R][S][Cin] inside the arena (it is the B operand of the implicit-GEMM
    convolution as stored — ops/conv.py), everything else is plain row-major."""
    n = param.numel()
    seg = flat[lo: lo + n]
    if param.dim() == 4 and not param.is_contiguous() and \
            param.is_contiguous(memory_format=torch.channels_last):
        return seg.as_strided(param.shape, param.stride())
    return seg.view(param.shape)


def _classify(opt) -> Optional[str]:
    """Return 'sgd' | 'adam' | 'adamw' if the wrapped optimizer's update rule is one the fused
    epilogue implements exactly, else None."""
    if isinstance(opt, torch.optim.SGD):
        return "sgd"
    if isinstance(opt, torch.optim.AdamW):
        kind = "adamw"
    elif isinstance(opt, torch.optim.Adam):
        kind = "adam"
    else:
        return None
    for g in opt.param_groups:
        if g.get("amsgrad", False) or g.get("differentiable", False):
            return None
    return kind


class FusedEngine:
    fuses_update = True

    @staticmethod
    def try_create(opt, buckets: List[Bucket], wire_dtype) -> Optional["FusedEngine"]:
        rt = _state.runtime()
        kind = _classify(opt)
        ok_dtypes = all(b.dtype in (torch.float32, torch.bfloat16, torch.float16) for b in buckets)
        devs = {b.device for b in buckets}
        wire_ok = wire_dtype is None or (wire_dtype in (torch.bfloat16, torch.float16) and
                                         all(b.dtype == torch.float32 for b in buckets))
        local_ok = kind is not None and ok_dtypes and len(devs) == 1 and wire_ok
        if rt.size > 1:
            votes = [None] * rt.size
            dist.all_gather_object(votes, bool(local_ok), group=rt.cpu_group)
            if not all(votes):
                return None
            symm = _state.get_symm()
            if symm is None:
                return None
        else:
            if not local_ok:
                return None
            from ..runtime.local import LocalRuntime
            symm = LocalRuntime.get()
            if symm is None:
                return None
        return FusedEngine(opt, buckets, symm, kind, wire_dtype)

    # ------------------------------------------------------------------ construction
    def __init__(self, opt, buckets: List[Bucket], symm, kind: str, wire_dtype=None):
        from ..runtime import symm as S
        self.S = S
        self.opt, self.buckets, self.symm, self.kind = weakref.proxy(opt), buckets, symm, kind
        self.device = buckets[0].device
        self.world = symm.world
        self.average = getattr(opt, "_op").name == "Average"
        # Wire compression (hvd.Compression.bf16 / fp16 with fp32 parameters): gradients cross NVLink in
        # the 16-bit wire dtype, the sum / scale / optimizer update run in fp32 inside the SAME fused
        # kernel, on the model's own fp32 parameters (they are the kernel's "master" copy).  Every rank
        # reduces the whole bucket (one-shot, fixed rank order) so all replicas apply the identical fp32
        # update; the only extra work vs the uncompressed path is ONE cast pass per bucket
        # (fp32 gradient -> wire dtype into symmetric memory), Horovod's `compress` step.
        self.wire = wire_dtype
        # Average with gradient_predivide_factor f: local gradients are scaled by 1/f BEFORE they are cast to
        # the wire dtype (keeps fp16 in range), the fused kernel applies f/N after the fp32 sum.  Without
        # wire compression the sum is fp32 end to end and (1/f)(f/N) == 1/N exactly, so nothing changes.
        self.predivide = float(getattr(opt, "_gradient_predivide_factor", 1.0) or 1.0)
        self.arenas: Dict[torch.dtype, dict] = {}
        for (dtype, device), n in arena_sizes(buckets).items():
            if self.wire is not None:
                wes = torch.empty((), dtype=self.wire).element_size()
                G = symm.alloc(n * wes)
                P = symm.alloc(n * wes)                     # 16-bit shadow of the updated parameters (kernel output)
                gw = G.tensor(self.wire, n)
                gw.zero_()
                P.tensor(self.wire, n).zero_()
                self.arenas[dtype] = {
                    "G": G, "P": P, "gw": gw,
                    "g": torch.zeros(n, dtype=torch.float32, device=device),      # local fp32 gradients (autograd)
                    "p": torch.zeros(n, dtype=torch.float32, device=device),      # the model's fp32 parameters
                    "M": None,
                    "S0": torch.zeros(n, dtype=torch.float32, device=device),
                    "S1": torch.zeros(n, dtype=torch.float32, device=device) if kind != "sgd" else None,
                }
                continue
            es = torch.empty((), dtype=dtype).element_size()
            G = symm.alloc(n * es)
            P = symm.alloc(n * es)
            g, p = G.tensor(dtype, n), P.tensor(dtype, n)
            g.zero_()
            p.zero_()
            self.arenas[dtype] = {
                "G": G, "P": P, "g": g, "p": p,
                "M": torch.zeros(n, dtype=torch.float32, device=device)
                if dtype != torch.float32 else None,
                "S0": torch.zeros(n, dtype=torch.float32, device=device),
                "S1": torch.zeros(n, dtype=torch.float32, device=device) if kind != "sgd" else None,
            }
        # re-home parameters and gradients into the arenas
        with torch.no_grad():
            for b in buckets:
                ar = self.arenas[b.dtype]
                for s in b.slots:
                    self._rehome(ar, b, s, first=True)
        self.params_changed()
        nb = len(buckets)
        self.step_ctr = torch.zeros(nb, dtype=torch.int32, device=self.device)
        self.ticket = torch.zeros(nb, dtype=torch.int32, device=self.device)
        self.lr_scale: Optional[torch.Tensor] = None
        self.side = torch.cuda.Stream(device=self.device, priority=-1)
        self._args: Dict[int, object] = {}
        self._algo: Dict[int, int] = {}
        for b in buckets:
            self._args[b.index], self._algo[b.index] = self._make_args(b)
        self._done = torch.cuda.Event()
        self.steps = 0
        self.rehomed = 0
        self.kernel_launches = 0
        self._state_dirty = False
        torch.cuda.synchronize(self.device)
        if self.world > 1:
            dist.barrier(group=_state.runtime().cpu_group)
        _ENGINES.add(self)

    def _rehome(self, ar, b: Bucket, s, first: bool = False) -> bool:
        """Make ``param.data`` / ``param.grad`` alias their arena slots.  Returns True if anything
        had to be moved.  Called once at construction and re-checked at every bucket launch: code
        that runs AFTER the optimizer is wrapped can silently re-point parameter storage —
        ``model.to(device)`` on an ``nn.LSTM`` calls ``flatten_parameters()``, which ``set_()``s every
        weight into a fresh cuDNN buffer (reference order: app/torch_train.py:259 then :261) — and
        the kernels would then train the arena while the model reads the stale buffer."""
        lo = b.flat_offset + s.offset
        p = s.param
        es = p.element_size()
        moved = False
        want_p = ar["p"].data_ptr() + lo * es
        if first or p.data_ptr() != want_p:
            pv = arena_view(ar["p"], lo, p)
            pv.copy_(p.data)
            p.data = pv
            if ar["M"] is not None and not first:
                ar["M"][lo: lo + s.numel].copy_(ar["p"][lo: lo + s.numel])
            moved = True
        g = p.grad
        want_g = ar["g"].data_ptr() + lo * es
        if first or g is None or g.data_ptr() != want_g:
            gv = arena_view(ar["g"], lo, p)
            if g is not None:
                gv.copy_(g)
            elif not first:
                gv.zero_()
            p.grad = gv
            moved = True
        return moved

    def _check_homes(self, b: Bucket):
        ar = self.arenas[b.dtype]
        base_p, base_g = ar["p"].data_ptr(), ar["g"].data_ptr()
        es = ar["p"].element_size()
        for s in b.slots:
            off = (b.flat_offset + s.offset) * es
            g = s.param.grad
            if s.param.data_ptr() != base_p + off or g is None or g.data_ptr() != base_g + off:
                with torch.no_grad():
                    self._rehome(ar, b, s)
                self.rehomed += 1

    def _make_args(self, b: Bucket):
        S, symm = self.S, self.symm
        ar = self.arenas[b.dtype]
        kdtype = self.wire if self.wire is not None else b.dtype      # dtype the kernel moves over NVLink
        es = torch.empty((), dtype=kdtype).element_size()
        off = b.flat_offset * es
        nbytes = b.numel * es
        a = S.ARArgs()
        gp, pp = ar["G"].ptrs_at(off), ar["P"].ptrs_at(off)
        for r in range(self.world):
            a.inp[r], a.out[r] = gp[r], pp[r]
        both_mc = ar["G"].mc_ptr != 0 and ar["P"].mc_ptr != 0
        algo = symm.pick_algo(nbytes, need_mc=both_mc)
        if self.wire is not None:
            algo = S.ALGO_ONESHOT            # every rank must hold the full fp32 update (see __init__)
        if algo == S.ALGO_NVLS and not both_mc:
            algo = S.ALGO_TWOSHOT
        if algo == S.ALGO_NVLS:
            a.in_mc, a.out_mc = ar["G"].mc_ptr + off, ar["P"].mc_ptr + off
        f32 = 4 * b.flat_offset
        if self.wire is not None:
            a.master = ar["p"].data_ptr() + f32      # the fp32 parameters themselves
        else:
            a.master = ar["M"].data_ptr() + f32 if ar["M"] is not None else 0
        a.s0 = ar["S0"].data_ptr() + f32
        a.s1 = ar["S1"].data_ptr() + f32 if ar["S1"] is not None else 0
        a.step_ctr = self.step_ctr.data_ptr() + 4 * b.index
        a.ticket = self.ticket.data_ptr() + 4 * b.index
        a.n = b.numel
        a.scale = (1.0 / self.world) if self.average else 1.0
        if self.wire is not None and self.average and self.predivide != 1.0:
            a.scale = self.predivide / self.world
        a.channel = S.CH_ENGINE
        a.zero_input, a.copy_back = 1, 0
        return a, algo

    # ------------------------------------------------------------------ hot path
    def _fill_hyper(self, a, group: dict):
        S, h = self.S, a.h
        lr = group["lr"]
        h.lr = float(lr)
        h.weight_decay = float(group.get("weight_decay", 0.0))
        h.maximize = int(bool(group.get("maximize", False)))
        if self.kind == "sgd":
            h.kind = S.OPT_SGD
            h.momentum = float(group.get("momentum", 0.0))
            h.dampening = float(group.get("dampening", 0.0))
            h.nesterov = int(bool(group.get("nesterov", False)))
        else:
            h.kind = S.OPT_ADAM
            b1, b2 = group["betas"]
            h.beta1, h.beta2, h.eps = float(b1), float(b2), float(group["eps"])
            h.adamw = int(self.kind == "adamw" or bool(group.get("decoupled_weight_decay", False)))

    def launch(self, b: Bucket):
        """Called from the autograd hook when the last gradient of ``b`` has been produced."""
        self._check_homes(b)
        a = self._args[b.index]
        self._fill_hyper(a, self.opt.param_groups[b.group_index])
        a.lr_scale = self.lr_scale.data_ptr() if self.lr_scale is not None else 0
        if self.wire is not None:            # compress: fp32 gradients -> wire dtype in symmetric memory
            ar = self.arenas[b.dtype]
            lo, hi = b.flat_offset, b.flat_offset + b.numel
            if self.average and self.predivide != 1.0:
                torch.mul(ar["g"][lo:hi], 1.0 / self.predivide, out=ar["gw"][lo:hi])
            else:
                ar["gw"][lo:hi].copy_(ar["g"][lo:hi])
            ar["g"][lo:hi].zero_()
        cur = torch.cuda.current_stream(self.device)
        ev = torch.cuda.Event()
        ev.record(cur)
        self.side.wait_event(ev)
        tl = _state.runtime().timeline
        if tl is not None:
            s_ev, e_ev = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s_ev.record(self.side)
        if nvtx.enabled():
            nvtx.push(f"bucket.{b.index} FUSED_ALLREDUCE_{self.S.ALGO_NAMES[self._algo[b.index]].upper()} "
                      f"{b.nbytes / 2**20:.1f}MB")
        kdtype = self.wire if self.wire is not None else b.dtype
        kbytes = b.numel * torch.empty((), dtype=kdtype).element_size()
        self.symm.launch_allreduce(a, self._algo[b.index], kdtype, kbytes, self.side)
        nvtx.pop()
        self.kernel_launches += 1
        if tl is not None:
            e_ev.record(self.side)
            tl.cuda_span(f"bucket.{b.index}", "FUSED_ALLREDUCE_" +
                         self.S.ALGO_NAMES[self._algo[b.index]].upper(), s_ev, e_ev,
                         bytes=b.nbytes)
        return True

    def wait_all(self, launched):
        self._done.record(self.side)
        torch.cuda.current_stream(self.device).wait_event(self._done)
        self.symm.check_errors()

    def after_step(self):
        self.steps += 1
        self._state_dirty = True

    def zero_grad(self):
        """Gradients are zeroed by the kernel that consumed them (zero-on-consume)."""
        return

    # ------------------------------------------------------------------ state plumbing
    def params_changed(self):
        """Parameters were written from outside (broadcast_parameters / load_state_dict):
        refresh the fp32 master copies."""
        for ar in self.arenas.values():
            if ar["M"] is not None:
                ar["M"].copy_(ar["p"])

    def _sharded(self, b: Bucket) -> bool:
        return self._algo[b.index] != self.S.ALGO_ONESHOT and self.world > 1

    def export_state(self):
        """Materialise ``optimizer.state`` (torch layout) from the flat state arenas so
        ``state_dict()`` / checkpointing / ``broadcast_optimizer_state`` see the usual
        per-parameter entries.  State of sliced buckets is sharded across ranks; unowned
        slices are still zero, so a Sum-allreduce of the arena reassembles it — which makes
        this call a COLLECTIVE when world > 1 (every rank must call it, like FSDP's full optimizer
        state dict): ``sd = opt.state_dict()`` on all ranks, then ``if hvd.rank() == 0: save``."""
        torch.cuda.current_stream(self.device).wait_stream(self.side)
        # the device-side counters are authoritative (CUDA-graph replays do not run Python)
        steps_dev = int(self.step_ctr.max().item()) if self.step_ctr.numel() else 0
        self.steps = max(self.steps, steps_dev)
        if steps_dev == 0:
            return
        opt = self.opt
        for b in self.buckets:
            ar = self.arenas[b.dtype]
            lo, hi = b.flat_offset, b.flat_offset + b.numel
            s0 = ar["S0"][lo:hi].clone()
            s1 = ar["S1"][lo:hi].clone() if ar["S1"] is not None else None
            if self._sharded(b):
                self.symm.allreduce_(s0)
                if s1 is not None:
                    self.symm.allreduce_(s1)
            for s in b.slots:
                st = opt.state[s.param]
                v0 = arena_view(s0, s.offset, s.param)
                if self.kind == "sgd":
                    if opt.param_groups[b.group_index].get("momentum", 0.0) != 0.0:
                        st["momentum_buffer"] = v0
                else:
                    st["step"] = torch.tensor(float(steps_dev))
                    st["exp_avg"] = v0
                    st["exp_avg_sq"] = arena_view(s1, s.offset, s.param)
        self._state_dirty = False

    def import_state(self):
        """Inverse of ``export_state`` (after ``optimizer.load_state_dict``)."""
        opt = self.opt
        steps = 0
        for b in self.buckets:
            ar = self.arenas[b.dtype]
            for s in b.slots:
                st = opt.state.get(s.param, {})
                lo = b.flat_offset + s.offset
                if self.kind == "sgd":
                    mb = st.get("momentum_buffer")
                    if mb is not None:
                        arena_view(ar["S0"], lo, s.param).copy_(mb)
                        steps = max(steps, 1)
                else:
                    if "exp_avg" in st:
                        arena_view(ar["S0"], lo, s.param).copy_(st["exp_avg"])
                        arena_view(ar["S1"], lo, s.param).copy_(st["exp_avg_sq"])
                        steps = max(steps, int(float(st.get("step", 0))))
            if self._sharded(b):
                # keep only the owned slice (others must stay zero for export's Sum-gather)
                vec = 16 // torch.empty((), dtype=b.dtype).element_size()
                nvec = b.numel // vec
                per = (nvec + self.world - 1) // self.world
                rlo = min(self.symm.rank * per, nvec) * vec
                rhi = min(rlo + per * vec, b.numel)
                for key in ("S0", "S1"):
                    t = ar[key]
                    if t is None:
                        continue
                    seg = t[b.flat_offset: b.flat_offset + b.numel]
                    seg[:rlo].zero_()
                    seg[rhi:].zero_()
        self.steps = max(self.steps, steps) if steps else self.steps
        if steps:
            self.step_ctr.fill_(steps)
        self.params_changed()

    def release(self):
        """Detach the model from the symmetric arenas (parameters and gradients become ordinary
        device tensors holding the current values) and drop every arena view, so the runtime can unmap
        and release the memory (``hvd.shutdown()``)."""
        if getattr(self, "_released", False) or not hasattr(self.symm, "free"):
            return
        self._released = True
        try:
            torch.cuda.current_stream(self.device).wait_stream(self.side)
            torch.cuda.synchronize(self.device)
        except Exception:      # noqa: BLE001
            pass
        with torch.no_grad():
            for b in self.buckets:
                for s in b.slots:
                    p = s.param
                    p.data = p.data.clone(memory_format=torch.preserve_format)
                    if p.grad is not None:
                        p.grad = p.grad.clone(memory_format=torch.preserve_format)
        for ar in self.arenas.values():
            for key in ("G", "P"):
                buf = ar.get(key)
                if buf is not None and hasattr(self.symm, "free"):
                    try:
                        self.symm.free(buf)
                    except Exception:  # noqa: BLE001
                        pass
            ar["g"] = ar["p"] = ar["G"] = ar["P"] = None
            ar["gw"] = None
        self._args.clear()

    def algorithms(self) -> Dict[int, str]:
        return {i: self.S.ALGO_NAMES[a] for i, a in self._algo.items()}
