"""``hvd.DistributedOptimizer`` — gradient-averaging optimizer wrapper.

Parity target: Horovod's ``DistributedOptimizer`` as used at reference
app/torch_train.py:259 (semantics: SURVEY.md §2.3 A6).  The returned object **is-a**
instance of the wrapped optimizer's class (dynamic subclass) with the same
``param_groups`` / ``state``.

H100-first design (vs Horovod's per-tensor ``allreduce_async_`` + host ``synchronize``):

* static bucket plan (``parallel/buckets.py``); ``p.grad`` tensors are views into flat
  buckets, so there is no pack/unpack;
* ``register_post_accumulate_grad_hook`` decrements a per-bucket counter; the bucket that
  completes is launched immediately on a high-priority **side stream** ordered after the
  backward stream by a CUDA event, overlapping communication with the rest of backward;
* on CUDA with the symmetric-memory runtime the bucket kernel is ONE sm_90a kernel that
  reduces across peers over NVLink (one-shot / two-shot / NVLS multicast, picked per
  bucket size), applies ``1/N`` (+ ``gradient_predivide_factor``), casts, and performs
  the SGD-momentum / Adam update in its epilogue (``parallel/fused_engine.py``;
  csrc/comm_kernels.cu) — ``step()`` is then just a stream wait, never a host wait;
* elsewhere (CPU/Gloo, NCCL fallback, unsupported optimizer) the bucket is all-reduced
  asynchronously and ``step()`` waits then calls the wrapped optimizer's ``step``.

When ``size() == 1`` no hooks are registered and the object behaves as the plain
optimizer (Horovod parity), unless ``B200DP_FUSED_SINGLE=1`` asks for the fused update
kernel on one GPU.
"""
from __future__ import annotations

import os
import warnings
from contextlib import contextmanager
from typing import Dict, List, Tuple

import torch
import torch.distributed as dist

from .. import _state
from ..utils import nvtx
from ..parallel.buckets import Bucket, plan_buckets, plan_hash, arena_sizes
from .compression import Compression
from . import mpi_ops
from .mpi_ops import Average, Sum, Adasum


class _DistributedOptimizer(torch.optim.Optimizer):
    # NOTE: methods of this class are copied into a dynamic subclass of the user's
    # optimizer class by ``DistributedOptimizer`` below.

    def __init__(self, params, named_parameters, compression, backward_passes_per_step, op,
                 gradient_predivide_factor, groups, num_groups, sparse_as_dense, process_set,
                 bucket_bytes, fused):
        super(self.__class__, self).__init__(params)
        self._compression = compression
        self._op = op
        self._process_set = process_set
        self._sparse_as_dense = sparse_as_dense
        self._gradient_predivide_factor = float(gradient_predivide_factor)
        self.backward_passes_per_step = int(backward_passes_per_step)
        self._should_synchronize = True
        self._synchronized = False
        self._hook_handles = []
        self._engine = None
        self._buckets: List[Bucket] = []
        self._flat: Dict[Tuple, torch.Tensor] = {}

        all_params = [p for g in self.param_groups for p in g["params"]]
        if named_parameters is not None:
            named_parameters = list(named_parameters)
        else:
            named_parameters = [(f"allreduce.noname.{gi}.{pi}", p)
                                for gi, g in enumerate(self.param_groups)
                                for pi, p in enumerate(g["params"])]
        if any(not isinstance(t, tuple) or len(t) != 2 for t in named_parameters):
            raise ValueError("named_parameters should be a sequence of tuples (name, parameter), "
                             "usually produced by model.named_parameters().")
        names = [n for n, _ in named_parameters]
        dups = sorted({n for n in names if names.count(n) > 1})
        if dups:
            raise ValueError("Parameter names in named_parameters must be unique. "
                             "Found duplicates: %s" % ", ".join(dups))
        named_ids = {id(p) for _, p in named_parameters}
        unnamed = [p for p in all_params if id(p) not in named_ids]
        if unnamed:
            raise ValueError("named_parameters was specified, but one or more model parameters "
                             "were not named. Python object ids: "
                             + ", ".join(str(id(p)) for p in unnamed))
        opt_ids = {id(p) for p in all_params}
        self._named = [(n, p) for n, p in named_parameters if id(p) in opt_ids]
        self._name_of = {id(p): n for n, p in self._named}
        self._group_of = {id(p): gi for gi, g in enumerate(self.param_groups)
                          for p in g["params"]}
        self._explicit_groups = groups
        self._num_groups = num_groups
        self._bucket_bytes = bucket_bytes
        self._fused_request = fused

        rt = _state._require_init()
        self._world = mpi_ops._ps_size(process_set)
        self._active = self._world > 1 or os.environ.get("B200DP_FUSED_SINGLE", "0") == "1"
        if self._active:
            self._setup()

    # ------------------------------------------------------------------ setup
    def _setup(self):
        rt = _state.runtime()
        trainable = [(n, p) for n, p in self._named if p.requires_grad]
        wire = getattr(self._compression, "wire_dtype", None)
        self._buckets = plan_buckets(
            trainable, self._group_of, self._bucket_bytes, self._explicit_groups,
            self._num_groups, grad_dtype=None)
        self._bucket_of: Dict[int, Bucket] = {}
        for b in self._buckets:
            for s in b.slots:
                self._bucket_of[id(s.param)] = b
        # plan agreement check over the control plane (replaces Horovod's negotiation)
        if self._world > 1 and self._process_set is None:
            digest = plan_hash(self._buckets)
            all_d = [None] * rt.size
            dist.all_gather_object(all_d, digest, group=rt.cpu_group)
            if any(d != digest for d in all_d):
                bad = [i for i, d in enumerate(all_d) if d != all_d[0]]
                raise RuntimeError(
                    f"DistributedOptimizer: gradient bucket plan differs across ranks "
                    f"(ranks {bad} disagree with rank 0) — models are not identical.")

        # try the fused sm_90a engine first
        self._engine = None
        want_fused = self._fused_request
        on_cuda = all(b.device.type == "cuda" for b in self._buckets) and len(self._buckets) > 0
        if want_fused is None:
            want_fused = os.environ.get("B200DP_FUSED", "1") == "1"
        if want_fused and on_cuda and self._process_set is None and self._op in (Average, Sum):
            from ..parallel.fused_engine import FusedEngine
            self._engine = FusedEngine.try_create(self, self._buckets, wire)
            if self._engine is None and self._fused_request:
                raise RuntimeError("fused=True requested but the fused sm_90a engine is "
                                   "unavailable: " + str(_state.runtime().symm_failed))
        if self._engine is None:
            self._setup_generic()

        self._pending = {b.index: len(b.slots) for b in self._buckets}
        self._passes: Dict[int, int] = {id(s.param): 0 for b in self._buckets for s in b.slots}
        self._launched: Dict[int, object] = {}
        self._register_hooks()

    def _setup_generic(self):
        """Flat arenas in ordinary memory; grads become views (zero-initialised)."""
        for (dtype, device), n in arena_sizes(self._buckets).items():
            self._flat[(dtype, device)] = torch.zeros(n, dtype=dtype, device=device)
        for b in self._buckets:
            flat = self._flat[(b.dtype, b.device)]
            for s in b.slots:
                view = flat[b.flat_offset + s.offset: b.flat_offset + s.offset + s.numel]
                view = view.view_as(s.param)
                if s.param.grad is not None:
                    view.copy_(s.param.grad)
                s.param.grad = view
        self._side_stream = None
        if any(b.device.type == "cuda" for b in self._buckets):
            self._side_stream = torch.cuda.Stream(priority=-1)

    def _bucket_tensor(self, b: Bucket) -> torch.Tensor:
        flat = self._flat[(b.dtype, b.device)]
        return flat[b.flat_offset: b.flat_offset + b.numel]

    def _register_hooks(self):
        from ..ops.grad_sink import ParamSink
        for b in self._buckets:
            for s in b.slots:
                hook = self._make_hook(s.param)
                h = s.param.register_post_accumulate_grad_hook(hook)
                self._hook_handles.append(h)
                if self._engine is not None:
                    # weight-gradient kernels may write straight into the bucket slot and then run the
                    # same bucket-ready logic autograd's AccumulateGrad would (ops/grad_sink.py)
                    s.param._b200dp_sink = ParamSink(
                        (lambda pid=id(s.param): self._passes[pid]),
                        (lambda p=s.param, hk=hook: hk(p)))

    # ------------------------------------------------------------------ hooks
    def _make_hook(self, p):
        pid = id(p)

        def hook(param):
            sink = getattr(param, "_b200dp_sink", None)
            if sink is not None:
                if sink.manual:            # the weight-gradient kernel already reported this pass
                    sink.manual = False
                    return
                sink.reset()
            b = self._bucket_of[pid]
            if b.index in self._launched:
                raise AssertionError(
                    "Gradients were computed more than backward_passes_per_step times "
                    "before call to step(). Increase backward_passes_per_step to "
                    "accumulate gradients locally.")
            self._passes[pid] += 1
            if self._passes[pid] > self.backward_passes_per_step:
                raise AssertionError(
                    "Gradients were computed more than backward_passes_per_step times "
                    "before call to step(). Increase backward_passes_per_step to "
                    "accumulate gradients locally.")
            if self._passes[pid] == self.backward_passes_per_step:
                g = param.grad
                if g is not None and g.is_sparse:
                    raise NotImplementedError(
                        "sparse gradients are not supported by the bucketed H100 path; "
                        "pass sparse_as_dense=True and use dense embeddings")
                if self._engine is None:
                    self._ensure_view(b, param)
                self._pending[b.index] -= 1
                if self._pending[b.index] == 0:
                    self._launch_bucket(b)
        return hook

    def _ensure_view(self, b: Bucket, param):
        """If the user replaced ``p.grad`` (e.g. zero_grad(set_to_none=True) from a foreign
        code path), re-attach it to the bucket view, copying the fresh gradient in."""
        flat = self._flat[(b.dtype, b.device)]
        for s in b.slots:
            if s.param is param:
                lo = b.flat_offset + s.offset
                if param.grad is None or param.grad.data_ptr() != flat[lo:lo + 1].data_ptr():
                    view = flat[lo: lo + s.numel].view_as(param)
                    if param.grad is not None:
                        view.copy_(param.grad)
                    else:
                        view.zero_()
                    param.grad = view
                return

    # ------------------------------------------------------------------ launch / sync
    def _launch_bucket(self, b: Bucket):
        tl = _state.runtime().timeline
        if tl is not None:
            tl.mark(f"bucket.{b.index}", "BUCKET_READY", bytes=b.nbytes, tensors=len(b.slots))
        if self._engine is not None:
            self._launched[b.index] = self._engine.launch(b)
            return
        t = self._bucket_tensor(b)
        div = self._gradient_predivide_factor
        prescale = 1.0 / div if div != 1.0 else 1.0
        postscale = div if div != 1.0 else 1.0
        if b.device.type == "cuda" and self._side_stream is not None:
            # order the collective after the gradients produced so far, on a side stream
            ev = torch.cuda.Event()
            ev.record(torch.cuda.current_stream(b.device))
            with torch.cuda.stream(self._side_stream):
                self._side_stream.wait_event(ev)
                h = self._launch_generic(t, prescale, postscale, b)
                done = torch.cuda.Event()
                done.record(self._side_stream)
            self._launched[b.index] = (h, done)
        else:
            self._launched[b.index] = (self._launch_generic(t, prescale, postscale, b), None)

    def _launch_generic(self, t, prescale, postscale, b: Bucket):
        wire = getattr(self._compression, "wire_dtype", None)
        name = f"bucket.{b.index}"
        if wire is not None and t.dtype != wire and t.dtype.is_floating_point:
            w = t.to(wire)
            h = mpi_ops.allreduce_async_(w, name=name, op=self._op, prescale_factor=prescale,
                                         postscale_factor=postscale,
                                         process_set=self._process_set, _lane=1)
            return ("cast", h, w, t)
        h = mpi_ops.allreduce_async_(t, name=name, op=self._op, prescale_factor=prescale,
                                     postscale_factor=postscale, process_set=self._process_set, _lane=1)
        return ("plain", h, None, t)

    def synchronize(self):
        """Complete all outstanding bucket reductions (launching buckets whose hooks never
        fired — unused parameters — with their current, possibly zero, gradients)."""
        if not self._active:
            self._synchronized = True
            return
        for b in self._buckets:
            if b.index not in self._launched:
                if self._engine is None:
                    for s in b.slots:
                        self._ensure_view(b, s.param)
                self._launch_bucket(b)
        if self._engine is not None:
            self._engine.wait_all(self._launched)
        else:
            for idx, (h, done) in list(self._launched.items()):
                kind, handle, w, t = h
                if done is not None:
                    with torch.cuda.stream(self._side_stream):
                        out = mpi_ops.synchronize(handle)
                        if kind == "cast":
                            t.copy_(out)
                        fin = torch.cuda.Event()
                        fin.record(self._side_stream)
                    torch.cuda.current_stream(t.device).wait_event(fin)
                else:
                    out = mpi_ops.synchronize(handle)
                    if kind == "cast":
                        t.copy_(out)
        self._launched.clear()
        for b in self._buckets:
            self._pending[b.index] = len(b.slots)
            if self._engine is not None:
                for s in b.slots:
                    sink = getattr(s.param, "_b200dp_sink", None)
                    if sink is not None:
                        sink.reset_step()
        for k in self._passes:
            self._passes[k] = 0
        self._synchronized = True

    @contextmanager
    def skip_synchronize(self):
        """``optimizer.synchronize(); clip; with optimizer.skip_synchronize(): optimizer.step()``"""
        self._should_synchronize = False
        try:
            yield
        finally:
            self._should_synchronize = True

    def set_backward_passes_per_step(self, passes: int):
        self.backward_passes_per_step = int(passes)
        if self._active:
            for k in self._passes:
                self._passes[k] = 0

    # ------------------------------------------------------------------ step / zero_grad
    def step(self, closure=None):
        if not self._active:
            return super(self.__class__, self).step(closure)
        tl = _state.runtime().timeline
        if tl is None:
            with nvtx.range("optimizer.step"):
                return self._step_impl(closure)
        tl.begin("optimizer", "STEP")
        try:
            return self._step_impl(closure)
        finally:
            tl.end("optimizer", "STEP")

    def _step_impl(self, closure=None):
        if self._engine is not None and self._engine.fuses_update:
            # The reduction kernels ARE the update.  step() therefore only has to make sure every
            # bucket has been launched exactly once for this iteration and order the stream.
            if not self._should_synchronize:
                raise RuntimeError(
                    "skip_synchronize() requires the un-fused path: construct "
                    "DistributedOptimizer(..., fused=False) when gradients must be modified "
                    "(e.g. clipped) between synchronize() and step().")
            loss = None
            if closure is not None:
                with torch.enable_grad():
                    loss = closure()
            if not self._synchronized:        # an explicit synchronize() already applied the update
                self.synchronize()
            self._synchronized = False
            self._engine.after_step()
            return loss
        if self._should_synchronize:
            if self._synchronized:
                warnings.warn("optimizer.step() called without optimizer.skip_synchronize() "
                              "context after optimizer.synchronize(). This can cause training "
                              "slowdown. You may want to consider using "
                              "optimizer.skip_synchronize() context if you use "
                              "optimizer.synchronize() in your code.")
            self.synchronize()
        self._synchronized = False
        return super(self.__class__, self).step(closure)

    def zero_grad(self, set_to_none: bool = True):
        """At size 1 this is the wrapped optimizer's ``zero_grad``.  When active, gradients are
        views into the flat buckets: they are zeroed in place (one memset per arena, or
        zero-on-consume inside the fused kernel) and stay attached; ``set_to_none`` is moot."""
        if not self._active:
            return super(self.__class__, self).zero_grad(set_to_none=set_to_none)
        if self._launched:
            raise AssertionError(
                "optimizer.zero_grad() was called after loss.backward() but before "
                "optimizer.step() or optimizer.synchronize(). This is prohibited as it can "
                "cause a race condition.")
        if self._engine is not None:
            self._engine.zero_grad()
            return
        # grads are bucket views: one memset per arena, views stay attached
        for flat in self._flat.values():
            flat.zero_()
        for b in self._buckets:
            for s in b.slots:
                if s.param.grad is None:
                    self._ensure_view(b, s.param)

    # ------------------------------------------------------------------ checkpoint / resume
    def state_dict(self):
        """Same layout as the wrapped optimizer's ``state_dict()``.  With the fused engine the
        momentum / Adam moments live in flat fp32 arenas (sharded by slice for the two-shot/NVLS
        buckets); they are gathered and exposed as ordinary per-parameter entries first.  With
        world > 1 this gather is a COLLECTIVE: call ``state_dict()`` on every rank, then let rank 0
        write the file (SURVEY.md §5.4: "rank 0 saves, then broadcast on resume")."""
        if self._engine is not None:
            from .mpi_ops import HorovodInternalError
            try:
                self._engine.export_state()
            except HorovodInternalError as e:
                raise HorovodInternalError(
                    str(e) + "  [optimizer.state_dict() is a collective when the fused engine "
                    "shards optimizer state across ranks: call it on EVERY rank, then save on "
                    "rank 0]") from e
        return super(self.__class__, self).state_dict()

    def load_state_dict(self, state_dict):
        super(self.__class__, self).load_state_dict(state_dict)
        if self._engine is not None:
            self._engine.import_state()

    # ------------------------------------------------------------------ misc
    @property
    def fused_engine(self):
        return self._engine

    def bucket_plan(self) -> List[Bucket]:
        return list(self._buckets)

    def remove_hooks(self):
        for h in self._hook_handles:
            h.remove()
        self._hook_handles.clear()
        for b in self._buckets:
            for s in b.slots:
                if hasattr(s.param, "_b200dp_sink"):
                    del s.param._b200dp_sink


def DistributedOptimizer(optimizer, named_parameters=None, compression=Compression.none,
                         backward_passes_per_step=1, op=Average, gradient_predivide_factor=1.0,
                         num_groups=0, groups=None, sparse_as_dense=False, process_set=None,
                         bucket_bytes=None, fused=None):
    """Wrap ``optimizer`` so gradients are averaged across ranks before the update.

    Arguments follow Horovod (SURVEY.md §2.3 A6); ``bucket_bytes`` and ``fused`` are
    H100-runtime extensions (``fused=None`` → use the fused sm_90a kernel when the
    optimizer is plain SGD(-momentum) / Adam / AdamW on CUDA with the symmetric runtime).
    """
    if op is Adasum:
        raise NotImplementedError("op=Adasum is not supported; use Average or Sum.")
    if gradient_predivide_factor != 1.0 and op is not Average:
        raise ValueError("gradient_predivide_factor not supported with op != Average")
    if num_groups and groups is not None:
        raise ValueError("only one of num_groups / groups may be given")
    if groups is not None:
        if isinstance(groups, int):
            num_groups, groups = groups, None
        elif not (isinstance(groups, list) and all(isinstance(g, list) for g in groups)):
            raise ValueError("groups should be a non-negative integer or a list of lists "
                             "of torch.Tensor")
    body = dict(_DistributedOptimizer.__dict__)
    body.pop("__dict__", None)
    body.pop("__weakref__", None)
    cls = type(optimizer.__class__.__name__, (optimizer.__class__,), body)
    return cls(optimizer.param_groups, named_parameters, compression, backward_passes_per_step,
               op, gradient_predivide_factor, groups, num_groups, sparse_as_dense, process_set,
               bucket_bytes, fused)
