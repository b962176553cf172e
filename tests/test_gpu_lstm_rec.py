"""K5 persistent LSTM recurrence (csrc/lstm_rec_sm90.cu) vs PyTorch's LSTM in fp32 (cuDNN TF32 disabled
for the oracle): outputs, final state, and gradients of every input and parameter."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _kern():
    from distributed_torch_horovod_gcp_b200.ops import kernels
    assert kernels.has("lstm_recurrent"), "lstm_rec kernels missing from libb200dp_kernels.so"
    return kernels


@pytest.mark.parametrize("B,T,F", [(32, 10, 23), (7, 3, 23), (100, 10, 23), (64, 5, 8)])
def test_lstm_recurrent_fwd_bwd(B, T, F):
    k = _kern()
    torch.manual_seed(3)
    old = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    try:
        lstm = torch.nn.LSTM(F, 256, batch_first=True).cuda()
        x = torch.randn(B, T, F, device="cuda", requires_grad=True)
        h0 = torch.randn(1, B, 256, device="cuda", requires_grad=True)
        c0 = torch.randn(1, B, 256, device="cuda", requires_grad=True)
        seq_ref, (hT_ref, cT_ref) = lstm(x, (h0, c0))
        prm = [lstm.weight_ih_l0, lstm.weight_hh_l0, lstm.bias_ih_l0, lstm.bias_hh_l0]
        seq, (hT, cT) = k.lstm_recurrent(x, h0, c0, *prm)
        # tf32 operands (10-bit mantissa), fp32 accumulation
        torch.testing.assert_close(seq, seq_ref, rtol=3e-3, atol=3e-3)
        torch.testing.assert_close(hT, hT_ref, rtol=3e-3, atol=3e-3)
        torch.testing.assert_close(cT, cT_ref, rtol=3e-3, atol=3e-3)
        g = torch.randn_like(seq)
        gh, gc = torch.randn_like(hT), torch.randn_like(cT)
        ins = [x, h0, c0] + prm
        ref = torch.autograd.grad([seq_ref, hT_ref, cT_ref], ins, [g, gh, gc])
        got = torch.autograd.grad([seq, hT, cT], ins, [g, gh, gc])
        for name, a, b in zip(["x", "h0", "c0", "w_ih", "w_hh", "b_ih", "b_hh"], got, ref):
            err = (a - b).norm() / b.norm().clamp_min(1e-6)
            assert err < 5e-3, (name, float(err))
    finally:
        torch.backends.cudnn.allow_tf32 = old


def test_lstm_model_uses_k5_and_trains():
    """The reference model end to end: forward through K5 + K6, backward, finite gradients for all ten
    parameter tensors, and no cuDNN RNN call (the launch counters move instead)."""
    from distributed_torch_horovod_gcp_b200.models import LSTM
    from distributed_torch_horovod_gcp_b200.ops import counters
    _kern()
    torch.manual_seed(0)
    m = LSTM(n_features=23, window_size=10, output_size=1, h_size=256, device=torch.device("cuda"))
    x = torch.randn(32, 10, 23, device="cuda")
    y = torch.randn(32, 1, 1, device="cuda")
    c0 = counters.snapshot()
    loss = torch.nn.functional.mse_loss(m(x), y)
    loss.backward()
    c1 = counters.snapshot()
    assert c1.get("lstm_rec_fwd", 0) > c0.get("lstm_rec_fwd", 0)
    assert c1.get("lstm_rec_bwd", 0) > c0.get("lstm_rec_bwd", 0)
    for n, p in m.named_parameters():
        assert p.grad is not None and torch.isfinite(p.grad).all(), n
        assert p.grad.abs().sum() > 0, n
    # large-batch validation pass (the reference evaluates the whole test split in one batch)
    with torch.no_grad():
        out = m(torch.randn(2500, 10, 23, device="cuda"))
    assert out.shape == (2500, 1, 1) and torch.isfinite(out).all()
