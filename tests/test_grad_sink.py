"""CPU tests of the autograd hand-off protocol in ops/grad_sink.py (no kernels involved): the GradBox
producer/consumer ordering rules."""
import torch

from distributed_torch_horovod_gcp_b200.ops.grad_sink import GradBox


def test_gradbox_unarmed_producer_keeps_its_gradient():
    box = GradBox()
    g = torch.ones(3)
    assert not box.park(g)              # no consumer registered in forward -> return the gradient to autograd
    assert box.take() == (None, None)


def test_gradbox_park_then_take():
    box = GradBox()
    box.armed = True                    # consumer's forward
    g, m = torch.ones(3), torch.zeros(1, dtype=torch.uint8)
    assert box.park(g, m)
    assert not box.park(torch.zeros(3))     # a second producer must not overwrite a parked gradient
    got, mask = box.take()
    assert got is g and mask is m
    assert box.take() == (None, None)       # handed over exactly once
    assert box.consumed


def test_gradbox_consumer_first_means_no_parking():
    """Projection block: the downsample dgrad has no data dependency on conv1's dgrad; if conv1 ran first the
    producer must fall back to returning its gradient (autograd then adds the two)."""
    box = GradBox()
    box.armed = True
    assert box.take() == (None, None)       # consumer backward ran with nothing parked
    assert not box.park(torch.ones(2))


def test_gradbox_fresh_per_forward():
    a, b = GradBox(), GradBox()
    a.armed = True
    a.park(torch.ones(1))
    assert b.dres is None and not b.armed and not b.consumed and not b.want_mask and b.ext_mask is None

