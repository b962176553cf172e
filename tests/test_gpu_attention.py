"""wgmma flash attention (csrc/attn_sm90.cu) vs an fp32 PyTorch reference: forward and all three
gradients, for the ViT-B/16 shape, a multi-block sequence, short sequences and the strided
[B,S,H,64] layout the model uses."""
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


def _kern():
    from distributed_torch_horovod_gcp_b200.ops import kernels
    assert kernels.has("attention_fused"), "attention kernels missing from libb200dp_kernels.so"
    return kernels


def _rel(a, b):
    return ((a.float() - b.float()).norm() / b.float().norm().clamp_min(1e-6)).item()


def _ref(q, k, v):
    s = (q @ k.transpose(-1, -2)) / math.sqrt(q.shape[-1])
    return torch.softmax(s, dim=-1) @ v


@pytest.mark.parametrize("B,H,S", [(8, 12, 197), (2, 16, 1024), (3, 4, 64), (2, 2, 130), (1, 3, 17), (2, 4, 384)])
def test_attention_fwd_bwd(B, H, S):
    k = _kern()
    torch.manual_seed(1)
    q, kk, v = [(torch.randn(B, H, S, 64, device="cuda") * 0.7).to(torch.bfloat16).requires_grad_(True)
                for _ in range(3)]
    refs = [t.detach().float().requires_grad_(True) for t in (q, kk, v)]
    o = k.attention_fused(q, kk, v)
    orf = _ref(*refs)
    assert o.shape == orf.shape
    assert _rel(o, orf) < 1.5e-2
    g = torch.randn(B, H, S, 64, device="cuda").to(torch.bfloat16)
    o.backward(g)
    orf.backward(g.float())
    for name, t, r in zip("qkv", (q, kk, v), refs):
        assert _rel(t.grad, r.grad) < 3e-2, (name, _rel(t.grad, r.grad))
    # second backward: the fp32 dQ workspace must have been re-zeroed
    for t in (q, kk, v):
        t.grad = None
    o2 = k.attention_fused(q, kk, v)
    o2.backward(g)
    assert _rel(q.grad, refs[0].grad) < 3e-2


def test_attention_model_layout_no_copies():
    """q, k, v as transposed views of [B*S, D] projection outputs; output reshapes to [B,S,D] as a view."""
    k = _kern()
    torch.manual_seed(2)
    B, S, H = 4, 197, 12
    mats = [(torch.randn(B * S, H * 64, device="cuda") * 0.5).to(torch.bfloat16) for _ in range(3)]
    q, kk, v = [m.view(B, S, H, 64).transpose(1, 2) for m in mats]
    o = k.attention_fused(q, kk, v)
    flat = o.transpose(1, 2).reshape(B, S, H * 64)
    assert flat.data_ptr() == o.data_ptr()                      # a view
    ref = _ref(q.float(), kk.float(), v.float()).transpose(1, 2).reshape(B, S, H * 64)
    assert _rel(flat, ref) < 1.5e-2


def test_vit_block_uses_attention_kernel():
    from distributed_torch_horovod_gcp_b200.models.vit import EncoderBlock
    from distributed_torch_horovod_gcp_b200.ops import counters
    _kern()
    torch.manual_seed(3)
    blk = EncoderBlock(768, 12, 3072).cuda().to(torch.bfloat16)
    x = (torch.randn(4, 197, 768, device="cuda") * 0.5).to(torch.bfloat16).requires_grad_(True)
    c0 = counters.snapshot()
    y = blk(x)
    y.float().mean().backward()
    c1 = counters.snapshot()
    assert c1.get("attn_fwd", 0) == c0.get("attn_fwd", 0) + 1
    assert c1.get("attn_bwd", 0) > c0.get("attn_bwd", 0)
    assert torch.isfinite(x.grad.float()).all()
