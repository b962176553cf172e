"""Direct-to-bucket weight gradients.

With the fused engine every ``param.grad`` is a view into a flat gradient bucket in symmetric
memory.  Autograd's ``AccumulateGrad`` then costs one ``add`` kernel (and often one layout
``copy``) per parameter per step — about 300 launches for ResNet-50.  A weight-gradient kernel that knows where the bucket slot is can
write there itself; this module is the handshake:

  forward  : ``note_forward(weight)``      (counts uses: shared weights keep the autograd path)
  backward : ``dst, accumulate, done = begin(weight)``
             ``dst is None`` -> return the gradient to autograd as usual;
             else write (``accumulate``: add to what is there) into ``dst`` — which IS
             ``weight.grad`` — call ``done()`` (runs the optimizer's bucket-ready hook) and return
             ``None`` to autograd for that input.

The sink object is installed on the parameter by ``DistributedOptimizer`` (torch/optimizer.py)
when the fused engine owns the gradients.
"""
from __future__ import annotations

import ctypes
import os
from typing import Callable, Optional, Tuple

import torch

_ENABLED = os.environ.get("B200DP_GRAD_SINK", "1") == "1"


class ParamSink:
    __slots__ = ("uses", "multi", "manual", "passes_done", "_fire")

    def __init__(self, passes_done: Callable[[], int], fire: Callable[[], None]):
        self.uses = 0
        self.multi = False
        self.manual = False                 # the kernel path already ran the bucket-ready logic
        self.passes_done = passes_done      # backward passes already accumulated in the slot
        self._fire = fire                   # the optimizer's post-accumulate hook for this param

    def fire(self):
        """Run the bucket-ready logic now.  Autograd still evaluates the parameter's AccumulateGrad
        node with an undefined gradient (no kernels) and — depending on the PyTorch version — calls
        the post-accumulate hook again; ``manual`` makes that second call a no-op."""
        self._fire()
        self.manual = True

    def reset(self):
        self.uses = 0
        self.multi = False

    def reset_step(self):
        self.reset()
        self.manual = False


def note_forward(weight) -> None:
    sink = getattr(weight, "_b200dp_sink", None)
    if sink is not None:
        sink.uses += 1
        if sink.uses > 1:
            sink.multi = True


def begin(weight, krsc: bool = False) -> Tuple[Optional[torch.Tensor], bool, Optional[Callable[[], None]]]:
    sink = getattr(weight, "_b200dp_sink", None)
    if not _ENABLED or sink is None or sink.multi or sink.uses != 1:
        return None, False, None
    g = weight.grad
    if g is None or g.dtype != weight.dtype or g.data_ptr() % 16:
        return None, False, None
    if krsc:
        if g.dim() != 4 or not g.is_contiguous(memory_format=torch.channels_last):
            return None, False, None
    elif not g.is_contiguous():
        if not (g.dim() == 4 and g.shape[2] == 1 and g.shape[3] == 1 and
                g.is_contiguous(memory_format=torch.channels_last)):
            return None, False, None
    return g, sink.passes_done() > 0, sink.fire


# ------------------------------------------------------------------ deferred fp32 -> grad-dtype casts
# Split-K weight-gradient kernels accumulate in a per-weight fp32 workspace that one pass converts into the
# gradient-bucket slot and re-zeroes.  With a sink, that pass is DEFERRED: records queue up here and one
# multi-tensor kernel converts all of them when the first bucket becomes ready (``flush_casts`` is called by
# the optimizer right before it launches a bucket's reduction, and by ``synchronize``).
class _CastSeg(ctypes.Structure):
    _fields_ = [("src", ctypes.c_void_p), ("dst", ctypes.c_void_p), ("n", ctypes.c_longlong),
                ("flags", ctypes.c_int), ("pad", ctypes.c_int)]


_pending_casts: list = []       # (device index, src ptr, dst ptr, n, flags, keep-alive tensors)
_DEFER = os.environ.get("B200DP_DEFER_CASTS", "1") == "1"


def defer_cast(lib, ws: torch.Tensor, dst: torch.Tensor, numel: int, acc: bool) -> bool:
    """Queue ``dst (+)= cast(ws); ws = 0``.  False when deferral is off / unsupported (caller casts now)."""
    if not _DEFER or not hasattr(lib, "b200dp_multi_cast_acc_zero") or numel % 4:
        return False
    flags = (1 if dst.dtype == torch.bfloat16 else 0) | (2 if acc else 0)
    if not _pending_casts:
        try:      # gradients must be complete when backward() returns, bucket launch or not
            torch.autograd.Variable._execution_engine.queue_callback(flush_casts)
        except RuntimeError:
            return False          # not inside a backward pass
    _pending_casts.append((lib, ws.device.index, ws.data_ptr(), dst.data_ptr(), numel, flags, (ws, dst)))
    return True


def flush_casts() -> None:
    if not _pending_casts:
        return
    by_dev = {}
    for rec in _pending_casts:
        by_dev.setdefault(rec[1], []).append(rec)
    _pending_casts.clear()
    for dev, recs in by_dev.items():
        lib = recs[0][0]
        arr = (_CastSeg * len(recs))()
        for i, (_, _, src, dst, n, flags, _keep) in enumerate(recs):
            arr[i].src, arr[i].dst, arr[i].n, arr[i].flags = src, dst, n, flags
        rc = lib.b200dp_multi_cast_acc_zero(ctypes.byref(arr), len(recs),
                                            torch.cuda.current_stream(dev).cuda_stream)
        if rc != 0:
            raise RuntimeError("multi_cast_acc_zero failed")
        from . import counters
        counters.bump("multi_cast_acc_zero")


class GradBox:
    """Hand-off of a residual-branch gradient between two autograd nodes of one block.

    In a residual block the block input ``x`` feeds the first convolution AND the skip connection, so
    autograd sums two activation-sized gradients with a stand-alone ``add`` kernel (16 of them per
    ResNet-50 step, ~1.1 ms).  With a box, the node that produces the skip gradient (the fused
    BN+add+ReLU backward) parks it here instead of returning it, and the first convolution's dgrad GEMM
    adds it in its epilogue (``C = A B + residual``) — the returned input gradient is already the sum.
    The consumer arms the box in ITS forward (which runs first), so a producer never withholds a
    gradient nobody will pick up; it marks the box ``consumed`` in its backward, so a producer that has
    no data dependency on the consumer (the downsample convolution of a projection block) only parks
    its gradient while the consumer is still to come.

    ``mask``: optional ReLU sign bits (1 byte / 8 channels) that the consumer's epilogue applies to
    ``dres`` — the BN+add+ReLU backward then parks the UNMASKED incoming gradient and does not write a
    masked copy at all.  ``ext_mask``: the same bits handed to the downsample BatchNorm of a projection
    block, whose incoming gradient is that unmasked tensor."""
    __slots__ = ("armed", "consumed", "dres", "mask", "ext_mask", "want_mask")

    def __init__(self):
        self.armed = False
        self.consumed = False
        self.want_mask = False       # the consumer is a BatchNorm backward that applies ``ext_mask`` to its dy
        self.dres = None
        self.mask = None
        self.ext_mask = None

    def park(self, grad, mask=None) -> bool:
        """Producer side: hand ``grad`` to the consumer if it is armed and still to run."""
        if not self.armed or self.consumed or self.dres is not None:
            return False
        self.dres, self.mask = grad, mask
        return True

    def take(self):
        """Consumer side (its backward): the parked (gradient, mask) or (None, None)."""
        self.consumed = True
        g, m = self.dres, self.mask
        self.dres = self.mask = None
        return g, m
