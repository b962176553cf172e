"""``functional.linear_cross_entropy`` and ``GPT.forward(idx, targets)`` on the CPU (the reference path)."""
import pytest
import torch
import torch.nn.functional as F

from distributed_torch_horovod_gcp_b200.models import gpt_tiny
from distributed_torch_horovod_gcp_b200.ops import functional as F2


def _inputs(N=37, D=24, V=50, seed=0, lead=None):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(N, D, generator=g)
    if lead is not None:
        x = x.view(*lead, D)
    w = torch.randn(V, D, generator=g) * 0.3
    t = torch.randint(0, V, (N,), generator=g)
    t[::5] = -100
    return x, w, t


@pytest.mark.parametrize("reduction", ["none", "sum", "mean"])
@pytest.mark.parametrize("ignore_index", [-100, 3])
def test_reference_is_the_torch_composition(reduction, ignore_index):
    x, w, t = _inputs(lead=(37,))
    t[t == -100] = ignore_index
    t[1] = 3
    xr, wr = x.clone().requires_grad_(True), w.clone().requires_grad_(True)
    xo, wo = x.clone().requires_grad_(True), w.clone().requires_grad_(True)
    got = F2.linear_cross_entropy(xr, wr, t, ignore_index=ignore_index, reduction=reduction)
    want = F.cross_entropy(F.linear(xo, wo).float(), t, ignore_index=ignore_index, reduction=reduction)
    assert got.dtype == torch.float32 and got.shape == want.shape
    assert torch.equal(got, want)
    gout = torch.linspace(0.5, 1.5, got.numel()).view(got.shape)
    got.backward(gout)
    want.backward(gout)
    assert torch.equal(xr.grad, xo.grad) and torch.equal(wr.grad, wo.grad)
    if reduction == "none":
        assert torch.equal(got[t == ignore_index], torch.zeros(int((t == ignore_index).sum())))


def test_reference_takes_leading_dimensions():
    x, w, t = _inputs(N=12, lead=(3, 4))
    got = F2.linear_cross_entropy(x, w, t.view(3, 4), reduction="none")
    want = F.cross_entropy(F.linear(x.reshape(12, -1), w), t, reduction="none")
    assert torch.equal(got, want)


def test_all_rows_ignored_mean_is_nan():
    x, w, t = _inputs(N=8)
    t[:] = -100
    assert torch.isnan(F2.linear_cross_entropy(x, w, t))
    assert float(F2.linear_cross_entropy(x, w, t, reduction="sum")) == 0.0


def test_invalid_arguments_raise_value_error():
    x, w, t = _inputs(N=8)
    with pytest.raises(ValueError):
        F2.linear_cross_entropy(x, w, t, reduction="avg")
    with pytest.raises(ValueError):
        F2.linear_cross_entropy(x, w, t[:7])
    with pytest.raises(ValueError):
        F2.linear_cross_entropy(x, w[:, :-1], t)


def test_gpt_forward_with_targets_is_the_loss_of_its_logits():
    torch.manual_seed(0)
    m = gpt_tiny()
    g = torch.Generator().manual_seed(1)
    idx = torch.randint(0, 512, (2, 16), generator=g)
    tgt = torch.randint(0, 512, (2, 16), generator=g)
    logits = m(idx)
    assert logits.shape == (32, 512)
    loss_ref = F.cross_entropy(logits, tgt.reshape(-1))
    loss = m(idx, tgt)
    assert loss.dim() == 0 and torch.equal(loss, loss_ref)
    assert torch.equal(m(idx, tgt.reshape(-1)), loss_ref)
    # the tied embedding's gradient sums both uses
    loss.backward()
    g1 = m.wte.weight.grad.clone()
    m.zero_grad()
    loss_ref = F.cross_entropy(m(idx), tgt.reshape(-1))
    loss_ref.backward()
    assert torch.equal(m.wte.weight.grad, g1)


def test_gpt_forward_without_targets_is_unchanged():
    torch.manual_seed(0)
    m = gpt_tiny()
    idx = torch.randint(0, 512, (2, 16))
    a = m(idx)
    b = m(idx, None)
    assert torch.equal(a, b)
