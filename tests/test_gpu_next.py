"""Acceptance tests for the 3x3 implicit-GEMM conv, attention and persistent LSTM kernels through their
`ops.kernels` entry points.  Each test skips until `ops.kernels.has(<name>)` turns true, so
wiring a new kernel into `ops/_bind.py` activates its numerics check automatically.

Expected entry points (all NHWC / bf16 unless noted):
  kernels.conv3x3(x, weight, stride)                     -> y          has("conv3x3")
  kernels.attention_fused(q, k, v)  [B,H,S,hd]           -> o          has("attention_fused")
  kernels.lstm_recurrent(x, h0, c0, w_ih, w_hh, b_ih, b_hh) fp32 -> (seq, (hT, cT))   has("lstm_recurrent")
"""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


def _kern(name):
    from distributed_torch_horovod_gcp_b200.ops import kernels
    if not kernels.has(name):
        pytest.skip(f"kernel '{name}' is not built")
    return kernels


def _rel(a, b):
    return ((a.float() - b.float()).norm() / b.float().norm().clamp_min(1e-6)).item()


@pytest.mark.parametrize("N,C,H,W,K,stride", [(8, 64, 56, 56, 64, 1), (4, 128, 28, 28, 128, 1),
                                              (4, 256, 28, 28, 256, 2), (2, 512, 7, 7, 512, 1)])
def test_conv3x3_matches_cudnn(N, C, H, W, K, stride):
    k = _kern("conv3x3")
    torch.manual_seed(0)
    x = torch.randn(N, C, H, W, device="cuda").to(torch.bfloat16).contiguous(
        memory_format=torch.channels_last).requires_grad_(True)
    w = (torch.randn(K, C, 3, 3, device="cuda") * 0.05).to(torch.bfloat16).contiguous(
        memory_format=torch.channels_last).requires_grad_(True)
    xr, wr = x.detach().float().requires_grad_(True), w.detach().float().requires_grad_(True)
    y = k.conv3x3(x, w, stride)
    yr = F.conv2d(xr, wr, None, stride, 1)
    assert y.shape == yr.shape and _rel(y, yr) < 8e-3
    g = torch.randn_like(y)
    y.backward(g)
    yr.backward(g.float())
    assert _rel(x.grad, xr.grad) < 1.5e-2 and _rel(w.grad, wr.grad) < 1.5e-2


@pytest.mark.parametrize("B,H,S,hd", [(8, 12, 197, 64), (2, 16, 1024, 64)])
def test_attention_matches_sdpa(B, H, S, hd):
    k = _kern("attention_fused")
    torch.manual_seed(1)
    q, kk, v = [(torch.randn(B, H, S, hd, device="cuda") * 0.5).to(torch.bfloat16).requires_grad_(True)
                for _ in range(3)]
    refs = [t.detach().float().requires_grad_(True) for t in (q, kk, v)]
    o = k.attention_fused(q, kk, v)
    orf = F.scaled_dot_product_attention(*refs)
    assert _rel(o, orf) < 1.5e-2
    g = torch.randn_like(o)
    o.backward(g)
    orf.backward(g.float())
    for t, r in zip((q, kk, v), refs):
        assert _rel(t.grad, r.grad) < 3e-2


def test_lstm_recurrent_matches_cudnn():
    k = _kern("lstm_recurrent")
    torch.manual_seed(2)
    lstm = torch.nn.LSTM(23, 256, batch_first=True).cuda()
    x = torch.randn(32, 10, 23, device="cuda", requires_grad=True)
    h0, c0 = torch.randn(1, 32, 256, device="cuda"), torch.randn(1, 32, 256, device="cuda")
    seq_ref, (hT_ref, cT_ref) = lstm(x, (h0, c0))
    seq, (hT, cT) = k.lstm_recurrent(x, h0, c0, lstm.weight_ih_l0, lstm.weight_hh_l0, lstm.bias_ih_l0,
                                     lstm.bias_hh_l0)
    # tf32 tensor cores are allowed (cuDNN's default): compare at 2e-3
    torch.testing.assert_close(seq, seq_ref, rtol=2e-3, atol=2e-3)
    torch.testing.assert_close(cT, cT_ref, rtol=2e-3, atol=2e-3)
    g = torch.randn_like(seq)
    gi_ref = torch.autograd.grad(seq_ref, [x, lstm.weight_hh_l0], g, retain_graph=True)
    gi = torch.autograd.grad(seq, [x, lstm.weight_hh_l0], g)
    for a, b in zip(gi, gi_ref):
        torch.testing.assert_close(a, b, rtol=5e-3, atol=5e-3)
