"""Bit-level pins of the ResNet bottleneck training path.

SHA-256 digests of what a bottleneck block (identity, projection stride 1, projection stride 2) computes in
one forward and backward, and of what three ResNet-50 steps through the fused optimizer compute, together
with the kernel-launch counts of one step.  The step is bit-reproducible (test_gpu_reductions.py), so equal
digests and equal counts mean the same kernels ran on the same inputs.  Grid sizes, and with them the
order of some sums, depend on the SM count, so the digests hold for the device they were recorded on."""
import hashlib
import json
import os

import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "bottleneck_sha256.json")

# name -> (inplanes, planes, stride, projection, H = W)
BLOCKS = {
    "identity": (256, 64, 1, False, 14),
    "projection_s1": (64, 64, 1, True, 28),
    "projection_s2": (256, 128, 2, True, 28),
}


def _sha(t: torch.Tensor) -> str:
    b = t.detach().cpu().contiguous().reshape(-1).view(torch.uint8)
    return hashlib.sha256(b.numpy().tobytes()).hexdigest()


def _nhwc(t):
    return t.to(torch.bfloat16).contiguous(memory_format=torch.channels_last)


def _device():
    p = torch.cuda.get_device_properties(0)
    return {"name": p.name, "sm_count": p.multi_processor_count}


def block_digests(kind: str) -> dict:
    from distributed_torch_horovod_gcp_b200.models.resnet import Bottleneck
    cin, planes, stride, proj, hw = BLOCKS[kind]
    torch.manual_seed(7)
    ds = nn.Sequential(nn.Conv2d(cin, planes * 4, 1, stride, bias=False), nn.BatchNorm2d(planes * 4)) \
        if proj else None
    blk = Bottleneck(cin, planes, stride, ds)
    with torch.no_grad():
        for m in blk.modules():
            if isinstance(m, nn.BatchNorm2d):
                m.weight.uniform_(0.5, 1.5)
                m.bias.uniform_(-0.2, 0.2)
    blk = blk.cuda().to(torch.bfloat16).to(memory_format=torch.channels_last).train()
    gen = torch.Generator(device="cuda").manual_seed(8)
    leaf = _nhwc(torch.randn(8, cin, hw, hw, device="cuda", generator=gen)).requires_grad_(True)
    x = leaf * 1.0                         # an intermediate, as in the network
    y = blk(x)
    g = _nhwc(torch.randn(y.shape, device="cuda", generator=gen))
    y.backward(g)
    torch.cuda.synchronize()
    out = {"out": _sha(y), "dx": _sha(leaf.grad)}
    out.update({"grad." + n: _sha(p.grad) for n, p in blk.named_parameters()})
    out.update({"buf." + n: _sha(b) for n, b in blk.named_buffers()})
    return out


def resnet_digests(hvd) -> dict:
    """As test_gpu_reductions.py::test_resnet_step_reproducible_in_one_process, with the grad sinks writing
    into the gradient buckets (``B200DP_FUSED_SINGLE=1`` must be set)."""
    from distributed_torch_horovod_gcp_b200.models import resnet50
    from distributed_torch_horovod_gcp_b200.ops import counters
    dev = torch.device("cuda", 0)
    gen = torch.Generator(device="cuda").manual_seed(11)
    batches = [(_nhwc(torch.randn(16, 3, 64, 64, device="cuda", generator=gen)),
                torch.randint(0, 100, (16,), device="cuda", generator=gen)) for _ in range(2)]
    torch.manual_seed(1234)
    model = resnet50(num_classes=100).to(dev).to(torch.bfloat16).to(memory_format=torch.channels_last)
    model.train()
    opt = hvd.DistributedOptimizer(torch.optim.SGD(model.parameters(), lr=0.1, momentum=0.9, weight_decay=1e-4),
                                   named_parameters=model.named_parameters())
    assert opt.fused_engine is not None
    losses = []
    for i in range(3):
        c0 = counters.snapshot()
        x, y = batches[i % 2]
        loss = F.cross_entropy(model(x).float(), y)
        loss.backward()
        opt.step()
        opt.zero_grad()
        losses.append(loss.detach().clone())
        c1 = counters.snapshot()
    torch.cuda.synchronize()
    opt.remove_hooks()
    h = hashlib.sha256()
    for k, v in model.state_dict().items():
        h.update(k.encode())
        h.update(_sha(v).encode())
    return {"loss": _sha(torch.stack(losses)), "state_dict": h.hexdigest(),
            "step_launches": {k: c1.get(k, 0) - c0.get(k, 0) for k in sorted(c1) if c1.get(k, 0) != c0.get(k, 0)}}


def record(hvd) -> dict:
    """The digests of this build, in the layout of ``GOLDEN``."""
    return {"device": _device(), "blocks": {k: block_digests(k) for k in BLOCKS},
            "resnet50": resnet_digests(hvd)}


def _golden():
    with open(GOLDEN) as f:
        gold = json.load(f)
    if gold["device"] != _device():
        pytest.skip(f"digests were recorded on {gold['device']}")
    return gold


@pytest.mark.parametrize("kind", list(BLOCKS))
def test_bottleneck_block_bits_unchanged(kind):
    want = _golden()["blocks"][kind]
    got = block_digests(kind)
    assert got.keys() == want.keys()
    differ = [k for k in want if got[k] != want[k]]
    assert not differ, f"differ: {differ}"


def test_resnet50_steps_bits_and_launches_unchanged(hvd_single, monkeypatch):
    monkeypatch.setenv("B200DP_FUSED_SINGLE", "1")
    want = _golden()["resnet50"]
    got = resnet_digests(hvd_single)
    assert got["step_launches"] == want["step_launches"]
    assert got["loss"] == want["loss"]
    assert got["state_dict"] == want["state_dict"]
