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
  R  fp32 reduced gradient | direction    local         clip mode (max_grad_norm=) and LARS / LAMB only

Clip mode (``max_grad_norm=``) splits each bucket's kernel in two phases, because a global norm needs
every bucket reduced before any bucket is updated: the bucket-ready hook launches a one-shot reduction
into R that also leaves one sum-of-squares slot per CTA (K1c); ``wait_all`` then launches one kernel
that folds all slots into the norm and the clip coefficient (K8) and one local update per bucket that
scales R by it and runs the unchanged K7 epilogue (K9).  One-shot everywhere means every rank holds the
same bits of R, so every rank computes the same norm without a further exchange.

LARS / LAMB (``hvd.LARS`` / ``hvd.LAMB``) scale each tensor's update by a trust ratio from norms over that
whole tensor, so their bucket kernel is split in two as well, but both phases run from the bucket's own hook
and still overlap backward: a one-shot reduction that writes the update direction to R and one fp32 partial
sum of squares of the master weights and of the direction per chunk (K10), then a local update that folds
each tensor's partials into its ratio in fp64 and applies it (K11).  A chunk is a fixed-size slice of one
tensor; the per-bucket chunk table is built once here and kept on the device, so graph replays reuse it.

Muon (``hvd.Muon``) follows each bucket's param group.  AdamW groups run the K7 launch with ``adamw=1``.  A Muon
bucket runs, from its own hook: a one-shot reduction that updates the momentum buffer (S0), writes u to R and one
fp32 sum of squares of u per chunk (K12); a local pass that folds each matrix's partials in fp64 and writes
X0 = bf16(u / max(‖u‖, eps)) into engine-owned scratch, transposed for tall matrices (K13); ``ns_steps``
Newton–Schulz iterations of three wgmma GEMMs per matrix (``ops.gemm.gemm``); and the update
w = w (1 - lr wd) - lr f O on the master weights (K14).  Every rank reduces the whole bucket and runs the same
deterministic GEMMs on the same bits of u, so the replicas stay bit-identical without exchanging O.
"""
from __future__ import annotations

import contextlib
import weakref
from typing import Dict, List, Optional

import torch
import torch.distributed as dist

from .. import _state
from ..utils import nvtx
from .buckets import Bucket, arena_sizes

_ENGINES: "weakref.WeakSet[FusedEngine]" = weakref.WeakSet()
LW_CHUNK_ELEMS = 16384          # elements per chunk of the LARS / LAMB partial norms
_LAYERWISE_KINDS = ("lars", "lamb")
_ONE_SHOT_ONLY_KINDS = ("lars", "lamb", "muon")    # kinds the engine does not combine with clipping or compression
_logged_layerwise_fallback = False
_logged_muon_fallback = False


def _elem_size(dtype: torch.dtype) -> int:
    return torch.empty((), dtype=dtype).element_size()


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


def _muon_unsupported(opt, buckets: List[Bucket]) -> Optional[str]:
    """Why the fused engine cannot run ``hvd.Muon`` ``opt`` on ``buckets``, or None: it needs the wgmma GEMM,
    fp32 / bf16 parameters and Muon matrices with both dimensions multiples of 8 (the GEMM's operand layouts)."""
    from ..ops import kernels
    if not (kernels.has("gemm") and kernels.has("gemm_scaled")):
        return "the kernels library with the wgmma GEMM and its scaled-residual entry point is not loaded"
    if any(b.dtype not in (torch.float32, torch.bfloat16) for b in buckets):
        return "parameters must be fp32 or bf16"
    for g in opt.param_groups:
        if g["use_muon"]:
            for p in g["params"]:
                if p.dim() != 2 or p.shape[0] % 8 or p.shape[1] % 8:
                    return f"a Muon matrix of shape {tuple(p.shape)} is not a multiple of 8 in both dimensions"
    return None


def _classify(opt) -> Optional[str]:
    """Return 'sgd' | 'adam' | 'adamw' | 'lars' | 'lamb' | 'muon' if the wrapped optimizer's update rule is one
    the fused kernels implement, else None."""
    from ..torch.optim import LARS, LAMB, Muon
    if isinstance(opt, Muon):
        return "muon"
    if isinstance(opt, torch.optim.SGD):
        return "sgd"
    if isinstance(opt, LARS):
        return "lars"
    if isinstance(opt, LAMB):
        return "lamb"
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
    def try_create(opt, buckets: List[Bucket], wire_dtype,
                   max_grad_norm: Optional[float] = None) -> Optional["FusedEngine"]:
        global _logged_layerwise_fallback, _logged_muon_fallback
        rt = _state.runtime()
        kind = _classify(opt)
        if kind in _ONE_SHOT_ONLY_KINDS and (wire_dtype is not None or max_grad_norm is not None):
            if not _logged_layerwise_fallback:
                _state.log.warning("%s with %s runs on the generic path (all-reduce, then the optimizer's own "
                                   "step): the fused engine does not combine them", type(opt).__name__,
                                   "max_grad_norm" if max_grad_norm is not None else "wire compression")
                _logged_layerwise_fallback = True
            kind = None
        if kind == "muon":
            why = _muon_unsupported(opt, buckets)
            if why is not None:
                if not _logged_muon_fallback:
                    _state.log.warning("Muon runs on the generic path (all-reduce, then the optimizer's own step): %s",
                                       why)
                    _logged_muon_fallback = True
                kind = None
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
        return FusedEngine(opt, buckets, symm, kind, wire_dtype, max_grad_norm)

    # ------------------------------------------------------------------ construction
    def __init__(self, opt, buckets: List[Bucket], symm, kind: str, wire_dtype=None,
                 max_grad_norm: Optional[float] = None):
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
        self.max_grad_norm = None if max_grad_norm is None else float(max_grad_norm)
        self.clip = self.max_grad_norm is not None
        self.layerwise = kind in _LAYERWISE_KINDS
        self.muon = kind == "muon"
        second_moment = kind in ("adam", "adamw", "lamb", "muon")
        self.arenas: Dict[torch.dtype, dict] = {}
        for (dtype, device), n in arena_sizes(buckets).items():
            def f32(on: bool = True):
                return torch.zeros(n, dtype=torch.float32, device=device) if on else None
            kdtype = self.wire if self.wire is not None else dtype      # dtype the kernel moves over NVLink
            G = symm.alloc(n * _elem_size(kdtype))
            P = symm.alloc(n * _elem_size(kdtype))                       # with wire: 16-bit shadow of the parameters
            g, p = G.tensor(kdtype, n), P.tensor(kdtype, n)
            g.zero_()
            p.zero_()
            ar = {"G": G, "P": P, "g": g, "p": p, "M": f32(dtype != torch.float32), "S0": f32(),
                  "S1": f32(second_moment), "R": f32(self.clip or self.layerwise or self.muon)}
            if self.wire is not None:       # local fp32 gradients (autograd) and the model's fp32 parameters
                ar["gw"], ar["g"], ar["p"] = g, f32(), f32()
            self.arenas[dtype] = ar
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
        self._kdtype: Dict[int, torch.dtype] = {}       # per bucket: dtype and byte count the kernel moves
        self._kbytes: Dict[int, int] = {}
        for b in buckets:
            self._kdtype[b.index] = self.wire if self.wire is not None else b.dtype
            self._kbytes[b.index] = b.numel * _elem_size(self._kdtype[b.index])
            self._args[b.index], self._algo[b.index] = self._make_args(b)
        self.grad_norm: Optional[torch.Tensor] = None
        if self.clip:
            # per-bucket slots of the reduce phase; a bucket's grid never changes, so slots past it stay 0
            self.slots = torch.zeros(nb * S.MAX_BLOCKS, dtype=torch.float32, device=self.device)
            self.grad_norm = torch.zeros((), dtype=torch.float32, device=self.device)
            self.coef = torch.ones((), dtype=torch.float32, device=self.device)
            self._clip_args: Dict[int, object] = {}
            self._apply_args: Dict[int, object] = {}
            for b in buckets:
                self._clip_args[b.index], self._apply_args[b.index] = self._make_clip_args(b)
            fin = S.ClipArgs()
            fin.slots, fin.nslots = self.slots.data_ptr(), self.slots.numel()
            fin.norm, fin.coef, fin.max_norm = self.grad_norm.data_ptr(), self.coef.data_ptr(), self.max_grad_norm
            self._fin_args = fin
        if self.layerwise or self.muon:
            self._build_chunks()
        if self.muon:
            self._build_muon()
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
        nbytes = self._kbytes[b.index]
        off = b.flat_offset * _elem_size(self._kdtype[b.index])
        a = S.ARArgs()
        gp, pp = ar["G"].ptrs_at(off), ar["P"].ptrs_at(off)
        for r in range(self.world):
            a.inp[r], a.out[r] = gp[r], pp[r]
        both_mc = ar["G"].mc_ptr != 0 and ar["P"].mc_ptr != 0
        algo = symm.pick_algo(nbytes, need_mc=both_mc)
        if self.wire is not None or self.clip or self.layerwise or self.muon:
            algo = S.ALGO_ONESHOT            # every rank must hold the full fp32 update / gradient (see __init__)
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

    def _make_clip_args(self, b: Bucket):
        """(reduce-phase ClipArgs, apply-phase ARArgs) of a bucket in clip mode.  The apply phase reads the
        already scaled R, so its ``scale`` is 1; everything else (outputs, master, state, step counter) is the
        bucket's ordinary one-shot argument block."""
        S, ar = self.S, self.arenas[b.dtype]
        k = S.ClipArgs()
        k.r = ar["R"].data_ptr() + 4 * b.flat_offset
        k.slots = self.slots.data_ptr() + 4 * S.MAX_BLOCKS * b.index
        k.norm, k.coef, k.max_norm = self.grad_norm.data_ptr(), self.coef.data_ptr(), self.max_grad_norm
        ap = S.ARArgs.from_buffer_copy(self._args[b.index])
        ap.scale = 1.0
        return k, ap

    def _build_chunks(self):
        """LARS / LAMB and Muon: in one pass over every bucket's slots, the chunk table (one device tensor, a slice
        per bucket) and, with Muon, the matrix of each chunk (``MuonMat`` rows, zero in AdamW buckets); then each
        bucket's ``ChunkArgs`` over its slices of the table, of the per-chunk partial sums and of R, embedded in its
        ``LwArgs`` (with its per-chunk ratio slots) or, in a Muon bucket, its ``MuonArgs``.  Tensors start on a
        16-byte boundary, so a vector never straddles two tensors; a tensor's last vector may end in padding, which
        is zero in every arena and adds nothing to either norm."""
        S = self.S
        rows, mats, first, span = [], [], {}, {}
        self._mu_mats = {}
        for b in self.buckets:
            vn = 16 // _elem_size(b.dtype)
            per = LW_CHUNK_ELEMS // vn
            base, use, x0, mm = len(rows), self._use_muon(b), 0, []
            for s in b.slots:
                v0, nv = s.offset // vn, (s.numel + vn - 1) // vn
                t0, cnt = len(rows) - base, (nv + per - 1) // per
                if cnt:
                    first[s.name] = len(rows)
                rows += [(v0 + c * per, min(per, nv - c * per), t0, cnt) for c in range(cnt)]
                shape = tuple(s.param.shape) if use else (0, 0)
                mats += [(*shape, s.offset, x0)] * cnt
                if use:
                    mm.append((*shape, x0))
                    x0 += s.numel
            self._mu_mats[b.index] = mm
            span[b.index] = (base, len(rows) - base)
        total = max(len(rows), 1)
        self.lw_chunks = torch.tensor(rows or [(0, 0, 0, 0)], dtype=torch.int32).to(self.device)
        self.lw_part = torch.zeros(2 * total, dtype=torch.float32, device=self.device)
        self.lw_ratio = torch.ones(total, dtype=torch.float32, device=self.device)
        if self.muon:
            self.mu_mats = torch.tensor(mats or [(0, 0, 0, 0)], dtype=torch.int32).to(self.device)
        self._lw_first = first
        self._lw_args: Dict[int, object] = {}
        self._mu_args: Dict[int, object] = {}
        for b in self.buckets:
            base, n = span[b.index]
            tab = S.ChunkArgs(r=self.arenas[b.dtype]["R"].data_ptr() + 4 * b.flat_offset,
                              part=self.lw_part.data_ptr() + 8 * base, chunks=self.lw_chunks.data_ptr() + 16 * base,
                              nchunks=n)
            if self.layerwise:
                self._lw_args[b.index] = S.LwArgs(tab=tab, ratio=self.lw_ratio.data_ptr() + 4 * base)
            elif self._use_muon(b):
                self._mu_args[b.index] = S.MuonArgs(tab=tab, mats=self.mu_mats.data_ptr() + 16 * base)

    def _build_muon(self):
        """Muon: the NS scratch, X0 / X1 (ping-pong operands, one region per matrix of the largest bucket) and the
        Gram G and its update H of the largest matrix, and each Muon bucket's NS input pointer."""
        x_elems = max([1] + [sum(r * c for r, c, _ in mm) for mm in self._mu_mats.values()])
        g_elems = max([1] + [min(r, c) ** 2 for mm in self._mu_mats.values() for r, c, _ in mm])
        bf = dict(dtype=torch.bfloat16, device=self.device)
        self.ns_x = [torch.zeros(x_elems, **bf), torch.zeros(x_elems, **bf)]
        self.ns_g, self.ns_h = torch.zeros(g_elems, **bf), torch.zeros(g_elems, **bf)
        for k in self._mu_args.values():
            k.x0 = self.ns_x[0].data_ptr()

    def _use_muon(self, b: Bucket) -> bool:
        return self.muon and bool(self.opt.param_groups[b.group_index]["use_muon"])

    def _newton_schulz(self, b: Bucket, group: dict) -> torch.Tensor:
        """``ns_steps`` iterations on every matrix of Muon bucket ``b``, from X0 in ``ns_x[0]``, on the current
        (side) stream: G = X Xᵀ, H = c G·G + b G, X ← a X + H·X.  Returns the scratch that holds O."""
        from ..ops import gemm as G
        a, bb, c = (float(v) for v in group["ns_coefficients"])
        steps = int(group["ns_steps"])
        for rows, cols, x0 in self._mu_mats[b.index]:
            p, q = min(rows, cols), max(rows, cols)
            gm, hm = self.ns_g[:p * p].view(p, p), self.ns_h[:p * p].view(p, p)
            splits = G._splits_for(p, p, q)
            for i in range(steps):
                x = self.ns_x[i % 2][x0: x0 + p * q].view(p, q)
                y = self.ns_x[(i + 1) % 2][x0: x0 + p * q].view(p, q)
                if splits > 1:
                    G.gemm(x, x, gm, p, p, q, out_mode=2, splits=splits)
                else:
                    G.gemm(x, x, gm, p, p, q)
                G.gemm(gm, gm, hm, p, p, p, b_mn=True, residual=gm, alpha=c, beta=bb)
                G.gemm(hm, x, y, p, q, p, b_mn=True, residual=x, beta=a)
                self.kernel_launches += 3
        return self.ns_x[steps % 2]

    def trust_ratios(self) -> Dict[str, torch.Tensor]:
        """LARS / LAMB: each parameter's trust ratio of the latest update, by name (0-dim fp32 views of a
        device buffer that every step, graph replays included, rewrites)."""
        if not self.layerwise:
            return {}
        return {name: self.lw_ratio[i] for name, i in self._lw_first.items()}

    # ------------------------------------------------------------------ hot path
    def _fill_hyper(self, a, group: dict):
        """This step's hyper-parameters of ``group`` and the ``lr_scale`` pointer, into argument block ``a``."""
        S, h = self.S, a.h
        a.lr_scale = self.lr_scale.data_ptr() if self.lr_scale is not None else 0
        lr = group["lr"]
        h.lr = float(lr)
        h.weight_decay = float(group.get("weight_decay", 0.0))
        h.maximize = int(bool(group.get("maximize", False)))
        if self.kind == "muon" and group["use_muon"]:
            h.kind = S.OPT_MUON
            h.momentum = float(group["momentum"])
            h.dampening = float(1 - group["momentum"])     # the lerp weight, formed in double as torch does
            h.nesterov = int(bool(group["nesterov"]))
        elif self.kind == "muon":
            h.kind, h.adamw = S.OPT_ADAM, 1
            b1, b2 = group["betas"]
            h.beta1, h.beta2, h.eps = float(b1), float(b2), float(group["adam_eps"])
        elif self.kind == "sgd":
            h.kind = S.OPT_SGD
            h.momentum = float(group.get("momentum", 0.0))
            h.dampening = float(group.get("dampening", 0.0))
            h.nesterov = int(bool(group.get("nesterov", False)))
        elif self.kind == "lars":
            h.kind = S.OPT_LARS
            h.momentum = float(group["momentum"])
        elif self.kind == "lamb":
            h.kind = S.OPT_LAMB
            b1, b2 = group["betas"]
            h.beta1, h.beta2, h.eps = float(b1), float(b2), float(group["eps"])
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
        op = "FUSED_ALLREDUCE_" + self.S.ALGO_NAMES[self._algo[b.index]].upper()
        kdtype, kbytes = self._kdtype[b.index], self._kbytes[b.index]
        with self._span(f"bucket.{b.index}", op, b.nbytes, f"bucket.{b.index} {op} {b.nbytes / 2**20:.1f}MB"):
            if self.clip:
                self.symm.launch_bucket("clip", a, self._clip_args[b.index], self.S.CLIP_REDUCE, kdtype, kbytes,
                                        self.side)
            elif self.muon and b.index in self._mu_args:
                self._launch_muon(b, a, kdtype, kbytes)
            elif self.layerwise:
                group = self.opt.param_groups[b.group_index]
                k = self._lw_args[b.index]
                k.adaptive = int(bool(group["adaptive"]))
                k.trust_coef = float(group["trust_coefficient"]) if self.kind == "lars" else 1.0
                self.symm.launch_bucket("lw", a, k, self.S.LW_REDUCE, kdtype, kbytes, self.side)
                self.symm.launch_bucket("lw", a, k, self.S.LW_APPLY, kdtype, kbytes, self.side)
                self.kernel_launches += 1
            else:
                self.symm.launch_allreduce(a, self._algo[b.index], kdtype, kbytes, self.side)
            self.kernel_launches += 1
        return True

    def _launch_muon(self, b: Bucket, a, kdtype, kbytes):
        """The four phases of a Muon bucket on the side stream: K12, K13, the NS GEMMs, K14."""
        S, group = self.S, self.opt.param_groups[b.group_index]
        k = self._mu_args[b.index]
        k.nesterov = int(bool(group["nesterov"]))
        k.lr_mode = 1 if group["adjust_lr_fn"] == "match_rms_adamw" else 0
        k.eps = float(group["eps"])
        self.symm.launch_bucket("muon", a, k, S.MUON_REDUCE, kdtype, kbytes, self.side)
        self.symm.launch_bucket("muon", a, k, S.MUON_NORMALIZE, kdtype, kbytes, self.side)
        with torch.cuda.stream(self.side):
            k.o = self._newton_schulz(b, group).data_ptr()
        self.symm.launch_bucket("muon", a, k, S.MUON_APPLY, kdtype, kbytes, self.side)
        self.kernel_launches += 2

    @contextlib.contextmanager
    def _span(self, name: str, op: str, nbytes: int, label: str):
        """NVTX range ``label`` and timeline span (``name``, ``op``) around the launches made inside it on the
        side stream."""
        tl = _state.runtime().timeline
        if tl is not None:
            s_ev, e_ev = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s_ev.record(self.side)
        nvtx.push(label)
        yield
        nvtx.pop()
        if tl is not None:
            e_ev.record(self.side)
            tl.cuda_span(name, op, s_ev, e_ev, bytes=nbytes)

    def wait_all(self, launched):
        if self.clip:
            self._clip_and_update()
        self._done.record(self.side)
        torch.cuda.current_stream(self.device).wait_event(self._done)
        self.symm.check_errors()

    def _clip_and_update(self):
        """Clip mode, after every bucket's reduce phase: the global norm and the clip coefficient (one
        launch), then the optimizer update of every bucket from R (one launch each), all on the side stream."""
        nbytes = sum(b.numel for b in self.buckets) * 4
        with self._span("optimizer", "CLIP_FINALIZE_APPLY", nbytes, "CLIP_FINALIZE_APPLY"):
            self.symm.launch_clip_finalize(self._fin_args, self.side)
            self.kernel_launches += 1
            for b in self.buckets:
                ap = self._apply_args[b.index]
                self._fill_hyper(ap, self.opt.param_groups[b.group_index])
                self.symm.launch_bucket("clip", ap, self._clip_args[b.index], self.S.CLIP_APPLY,
                                        self._kdtype[b.index], self._kbytes[b.index], self.side)
                self.kernel_launches += 1

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
                elif self.kind == "lars" or self._use_muon(b):
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
                if self.kind in ("sgd", "lars") or self._use_muon(b):
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
            ar["gw"] = ar["R"] = None
        self._args.clear()

    def algorithms(self) -> Dict[int, str]:
        return {i: self.S.ALGO_NAMES[a] for i, a in self._algo.items()}
