"""Stacked and bidirectional LSTMs on the K5 recurrence kernels (ops/lstm_rec.py::lstm_stack), against
PyTorch's LSTM in fp32 (cuDNN TF32 disabled for the oracle)."""
import hashlib
import json
import os

import pytest
import torch

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "lstm_rec_reference_shape_sha256.json")


def _kern():
    from distributed_torch_horovod_gcp_b200.ops import kernels
    assert kernels.has("lstm_recurrent"), "lstm_rec kernels missing from libb200dp_kernels.so"
    return kernels


def reference_shape_digests():
    """SHA-256 of every output and gradient of one ``lstm_recurrent`` call at the reference shape
    (B=32, T=10, F=23), on inputs drawn from a seeded CPU generator."""
    from distributed_torch_horovod_gcp_b200.ops import lstm_rec
    _kern()
    B, T, F, H = 32, 10, 23, 256
    g = torch.Generator().manual_seed(20261016)
    k = H ** -0.5

    def u(*shape):
        return ((torch.rand(*shape, generator=g) * 2 - 1) * k).cuda().requires_grad_()

    def n(*shape):
        return torch.randn(*shape, generator=g).cuda()

    w_ih, w_hh, b_ih, b_hh = u(4 * H, F), u(4 * H, H), u(4 * H), u(4 * H)
    x = n(B, T, F).requires_grad_()
    h0 = n(1, B, H).requires_grad_()
    c0 = n(1, B, H).requires_grad_()
    dseq, dhT, dcT = n(B, T, H), n(1, B, H), n(1, B, H)
    seq, (hT, cT) = lstm_rec.lstm_recurrent(x, h0, c0, w_ih, w_hh, b_ih, b_hh)
    dx, dh0, dc0, dw_ih, db_ih, db_hh = torch.autograd.grad(
        [seq, hT, cT], [x, h0, c0, w_ih, b_ih, b_hh], [dseq, dhT, dcT])
    out = {"seq": seq, "h_n": hT, "c_n": cT, "dx": dx, "dh0": dh0, "dc0": dc0, "dW_ih": dw_ih,
           "db_ih": db_ih, "db_hh": db_hh}
    return {name: hashlib.sha256(t.detach().contiguous().cpu().numpy().tobytes()).hexdigest()
            for name, t in out.items()}


def test_reference_shape_bits_unchanged():
    """The one-layer unidirectional F <= 32 path keeps its launches and arithmetic: outputs and gradients are
    bit-identical to the digests recorded before stacking and bidirectional layers were added (dW_hh is left
    out: it is summed with fp32 atomics)."""
    with open(GOLDEN) as f:
        want = json.load(f)
    assert reference_shape_digests() == want


def _oracle(F, L, D):
    return torch.nn.LSTM(F, 256, num_layers=L, bidirectional=D == 2, batch_first=True).cuda()


def _weights(lstm):
    return [w for ws in lstm.all_weights for w in ws]


def _rel(a, b):
    return float((a - b).norm() / b.norm().clamp_min(1e-6))


# (layers, directions, features, batch, steps): every value of each axis appears at least once
CASES = [(1, 1, 1, 1, 1), (1, 2, 23, 7, 3), (2, 1, 33, 32, 10), (2, 2, 64, 100, 3), (3, 2, 256, 7, 10),
         (3, 1, 512, 32, 3), (1, 2, 512, 1, 10), (2, 2, 23, 32, 10), (1, 1, 256, 100, 1)]


@pytest.mark.parametrize("L,D,F,B,T", CASES)
def test_lstm_stack_matches_nn_lstm(L, D, F, B, T):
    from distributed_torch_horovod_gcp_b200.ops import lstm_rec
    _kern()
    torch.manual_seed(5)
    old = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    try:
        lstm = _oracle(F, L, D)
        x = torch.randn(B, T, F, device="cuda", requires_grad=True)
        h0 = torch.randn(L * D, B, 256, device="cuda", requires_grad=True)
        c0 = torch.randn(L * D, B, 256, device="cuda", requires_grad=True)
        seq_ref, (hN_ref, cN_ref) = lstm(x, (h0, c0))
        assert lstm_rec.stack_supported(lstm, x)
        seq, (hN, cN) = lstm_rec.lstm_stack(x, h0, c0, _weights(lstm), L, D == 2)
        assert seq.shape == (B, T, D * 256) and hN.shape == cN.shape == (L * D, B, 256)
        # tf32 operands (10-bit mantissa), fp32 accumulation and state
        torch.testing.assert_close(seq, seq_ref, rtol=3e-3, atol=3e-3)
        torch.testing.assert_close(hN, hN_ref, rtol=3e-3, atol=3e-3)
        torch.testing.assert_close(cN, cN_ref, rtol=3e-3, atol=3e-3)
        g, gh, gc = torch.randn_like(seq), torch.randn_like(hN), torch.randn_like(cN)
        names = ["x", "h0", "c0"] + [n for ns in lstm._all_weights for n in ns]
        ins = [x, h0, c0] + _weights(lstm)
        ref = torch.autograd.grad([seq_ref, hN_ref, cN_ref], ins, [g, gh, gc])
        got = torch.autograd.grad([seq, hN, cN], ins, [g, gh, gc])
        for name, a, b in zip(names, got, ref):
            assert _rel(a, b) < 5e-3, (name, _rel(a, b))
    finally:
        torch.backends.cudnn.allow_tf32 = old


def test_stacked_bidirectional_model_runs_without_cudnn(monkeypatch):
    from distributed_torch_horovod_gcp_b200.models import LSTM
    from distributed_torch_horovod_gcp_b200.ops import counters
    _kern()
    torch.manual_seed(0)
    m = LSTM(23, 10, 1, 256, n_layers=2, bidirectional=True, device=torch.device("cuda"))

    def no_cudnn(*a, **k):
        raise AssertionError("cuDNN RNN called")
    monkeypatch.setattr(m.lstm, "forward", no_cudnn)
    x = torch.randn(32, 10, 23, device="cuda")
    y = torch.randn(32, 1, 1, device="cuda")
    c0 = counters.snapshot()
    torch.nn.functional.mse_loss(m(x), y).backward()
    c1 = counters.snapshot()
    assert c1.get("lstm_rec_fwd", 0) > c0.get("lstm_rec_fwd", 0)
    assert c1.get("lstm_rec_bwd", 0) > c0.get("lstm_rec_bwd", 0)
    for n, p in m.named_parameters():
        assert p.grad is not None and torch.isfinite(p.grad).all(), n
        assert p.grad.abs().sum() > 0, n
    with torch.no_grad():                    # the reference validates on the whole test split in one batch
        out = m(torch.randn(2500, 10, 23, device="cuda"))
    assert out.shape == (2500, 1, 1) and torch.isfinite(out).all()


def test_unsupported_shape_falls_back_to_cudnn():
    import copy
    from distributed_torch_horovod_gcp_b200.models import LSTM
    from distributed_torch_horovod_gcp_b200.ops import counters
    _kern()
    torch.manual_seed(0)
    m = LSTM(23, 10, 1, 128, device=torch.device("cuda"))
    ref = copy.deepcopy(m)
    ref._fused = False
    x = torch.randn(16, 10, 23, device="cuda")
    c0 = counters.snapshot()
    torch.manual_seed(1)
    out = m(x)
    c1 = counters.snapshot()
    torch.manual_seed(1)
    out_ref = ref(x)
    assert c1.get("lstm_rec_fwd", 0) == c0.get("lstm_rec_fwd", 0)
    torch.testing.assert_close(out, out_ref, rtol=1e-4, atol=1e-5)


def test_stacked_bidirectional_training_step(hvd_single, monkeypatch):
    """2-layer bidirectional model through hvd.DistributedOptimizer(Adam) with the fused engine: every
    weight gradient (the _reverse ones included) goes through its grad sink, one step matches a clone
    trained on the cuDNN path, and a CUDA-graphed step replays with the eager loss."""
    import copy
    monkeypatch.setenv("B200DP_FUSED_SINGLE", "1")
    hvd = hvd_single
    from distributed_torch_horovod_gcp_b200.models import LSTM
    from distributed_torch_horovod_gcp_b200.utils.graph import GraphedStep
    _kern()
    dev = torch.device("cuda", 0)
    torch.manual_seed(0)
    m = LSTM(23, 10, 1, 256, n_layers=2, bidirectional=True, device=dev)
    ref = copy.deepcopy(m)
    ref._fused = False
    B = 32
    h0 = torch.randn(4, B, 256, device=dev)
    c0 = torch.randn(4, B, 256, device=dev)
    for mod in (m, ref):                     # the same initial state for both models
        mod.init_hidden = lambda b: (h0, c0)
    lr = 1e-3
    opt = hvd.DistributedOptimizer(torch.optim.Adam(m.parameters(), lr=lr), named_parameters=m.named_parameters())
    assert opt.fused_engine is not None
    ropt = torch.optim.Adam(ref.parameters(), lr=lr)
    fired = set()
    for n, p in m.lstm.named_parameters():
        sink = getattr(p, "_b200dp_sink", None)
        assert sink is not None, n

        def rec(f=sink._fire, n=n):
            fired.add(n)
            f()
        sink._fire = rec
    x = torch.randn(B, 10, 23, device=dev)
    y = torch.randn(B, 1, 1, device=dev)
    before = [p.detach().clone() for p in m.parameters()]
    old = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    try:
        torch.nn.functional.mse_loss(m(x), y).backward()
        opt.step()
        opt.zero_grad()
        torch.nn.functional.mse_loss(ref(x), y).backward()
        ref_grads = [p.grad.detach().clone() for p in ref.parameters()]
        ropt.step()
        ropt.zero_grad()
    finally:
        torch.backends.cudnn.allow_tf32 = old
    torch.cuda.synchronize()
    assert fired == {n for n, _ in m.lstm.named_parameters()}
    assert any(n.endswith("_reverse") for n in fired)
    for (n, a), b, p0, g in zip(m.named_parameters(), ref.parameters(), before, ref_grads):
        # Adam's first step moves each element by lr * g / (|g| + eps), about lr * sign(g).  Where the gradient
        # is well above the two paths' difference (tf32 products: ~5e-3 of its norm) the updates must agree to
        # rounding; only elements near zero may take the other sign.
        da, db = a.detach() - p0, b.detach() - p0
        big = g.abs() > 0.1 * g.abs().mean()
        assert big.any(), n
        torch.testing.assert_close(da[big], db[big], rtol=1e-3, atol=1e-3 * lr, msg=lambda s: f"{n}: {s}")
        assert float((da - db).abs().mean()) < 0.02 * lr, (n, float((da - db).abs().mean()))

    def step(xb, yb):
        loss = torch.nn.functional.mse_loss(m(xb), yb)
        loss.backward()
        opt.step()
        opt.zero_grad()
        return loss.detach()
    graphed = GraphedStep(step, [x, y], warmup=2)
    with torch.no_grad():
        le = torch.nn.functional.mse_loss(m(x), y)
    lg = graphed(x, y)
    torch.cuda.synchronize()
    torch.testing.assert_close(lg, le, rtol=1e-6, atol=0)


if __name__ == "__main__":
    print(json.dumps(reference_shape_digests(), indent=1))
