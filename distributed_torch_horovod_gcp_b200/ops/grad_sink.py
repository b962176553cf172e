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
