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
    """Removed.  The name stays importable so that code written against the former cross-node hand-off of
    skip-connection gradients fails where it uses it, with this pointer, rather than at import."""

    def __init__(self, *args, **kwargs):
        raise RuntimeError("GradBox was removed: a ResNet bottleneck block runs as one autograd node "
                           "(ops/bottleneck.py) that adds the skip gradient in conv1's dgrad itself")
