"""Stacked LSTMs with inter-layer dropout on the K5 recurrence kernels (ops/lstm_rec.py::lstm_stack with
``dropout > 0``), against single-layer PyTorch LSTMs fed the same masks (cuDNN TF32 disabled for the oracle)."""
import hashlib
import json
import os

import pytest
import torch

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "lstm_stack_sha256.json")
# two stack cases of test_gpu_lstm_stack.py: together they run lstm_in_mma_kernel in all three modes
GOLDEN_CASES = [(2, 2, 23, 32, 10), (3, 1, 512, 32, 3)]


def _kern():
    from distributed_torch_horovod_gcp_b200.ops import kernels
    assert kernels.has("lstm_recurrent"), "lstm_rec kernels missing from libb200dp_kernels.so"
    return kernels


def stack_digests(L, D, F, B, T, **kw):
    """SHA-256 of every output and gradient of one ``lstm_stack`` call, on inputs drawn from a seeded CPU
    generator (``kw`` goes to ``lstm_stack``).  dW_hh is left out: it is summed with fp32 atomics."""
    from distributed_torch_horovod_gcp_b200.ops import lstm_rec
    _kern()
    H = 256
    g = torch.Generator().manual_seed(20261016 + 1000 * L + 100 * D + F)
    k = H ** -0.5

    def u(*shape):
        return ((torch.rand(*shape, generator=g) * 2 - 1) * k).cuda().requires_grad_()

    def n(*shape):
        return torch.randn(*shape, generator=g).cuda()

    weights, names = [], []
    for l in range(L):
        for d in range(D):
            sfx = f"_l{l}" + ("_reverse" if d else "")
            fin = F if l == 0 else D * H
            weights += [u(4 * H, fin), u(4 * H, H), u(4 * H), u(4 * H)]
            names += ["weight_ih" + sfx, "weight_hh" + sfx, "bias_ih" + sfx, "bias_hh" + sfx]
    x = n(B, T, F).requires_grad_()
    h0 = n(L * D, B, H).requires_grad_()
    c0 = n(L * D, B, H).requires_grad_()
    dseq, dhN, dcN = n(B, T, D * H), n(L * D, B, H), n(L * D, B, H)
    seq, (hN, cN) = lstm_rec.lstm_stack(x, h0, c0, weights, L, D == 2, **kw)
    keep = [i for i, nm in enumerate(names) if not nm.startswith("weight_hh")]
    grads = torch.autograd.grad([seq, hN, cN], [x, h0, c0] + [weights[i] for i in keep], [dseq, dhN, dcN])
    out = {"seq": seq, "h_n": hN, "c_n": cN, "dx": grads[0], "dh0": grads[1], "dc0": grads[2]}
    out.update({"d" + names[i]: gr for i, gr in zip(keep, grads[3:])})
    return {name: hashlib.sha256(t.detach().contiguous().cpu().numpy().tobytes()).hexdigest()
            for name, t in out.items()}


def _case_id(case):
    return "L{}_D{}_F{}_B{}_T{}".format(*case)


@pytest.mark.parametrize("case", GOLDEN_CASES, ids=_case_id)
def test_no_dropout_bits_unchanged(case):
    """p = 0, and p > 0 in eval mode, run the launches and arithmetic of the stack before dropout existed:
    outputs and gradients are bit-identical to digests recorded then."""
    with open(GOLDEN) as f:
        want = json.load(f)[_case_id(case)]
    assert stack_digests(*case, dropout=0.0) == want
    assert stack_digests(*case, dropout=0.5, training=False) == want


def _rel(a, b):
    return float((a - b).norm() / b.norm().clamp_min(1e-6))


def _oracle(lstm, L, D, p, x, h0, c0, keep):
    """Single-layer nn.LSTMs sharing ``lstm``'s parameters, each fed the layer below's output through the
    kernels' own keep mask."""
    inp, hs, cs = x, [], []
    for l in range(L):
        mod = torch.nn.LSTM(inp.shape[2], 256, bidirectional=D == 2, batch_first=True).cuda()
        for d in range(D):
            sfx = "_reverse" if d else ""
            for kind in ("weight_ih", "weight_hh", "bias_ih", "bias_hh"):
                setattr(mod, f"{kind}_l0{sfx}", getattr(lstm, f"{kind}_l{l}{sfx}"))
        out, (h, c) = mod(inp, (h0[l * D:(l + 1) * D], c0[l * D:(l + 1) * D]))
        hs.append(h)
        cs.append(c)
        if l < L - 1:
            inp = out * keep[l] / (1 - p) if p < 1 else torch.zeros_like(out)
    return out, torch.cat(hs), torch.cat(cs)


# (layers, directions, features, batch, steps, p): every value of each axis appears at least once
ORACLE_CASES = [(2, 1, 23, 1, 10, 0.5), (2, 2, 512, 7, 1, 0.1), (3, 2, 23, 32, 10, 1.0),
                (3, 1, 512, 100, 10, 0.5), (2, 2, 23, 100, 10, 0.1), (3, 2, 512, 7, 10, 0.5)]


@pytest.mark.parametrize("L,D,F,B,T,p", ORACLE_CASES)
def test_dropout_matches_masked_layerwise_lstm(L, D, F, B, T, p):
    """Training-mode dropout against one-layer PyTorch LSTMs fed ``seq * keep / (1 - p)`` with the kernels'
    mask; with two directions, both directions of the next layer read that one mask."""
    from distributed_torch_horovod_gcp_b200.ops import lstm_rec
    _kern()
    torch.manual_seed(7)
    old = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    try:
        lstm = torch.nn.LSTM(F, 256, num_layers=L, bidirectional=D == 2, batch_first=True, dropout=p).cuda()
        assert lstm_rec.stack_supported(lstm, torch.empty(B, T, F, device="cuda"))
        x = torch.randn(B, T, F, device="cuda", requires_grad=True)
        h0 = torch.randn(L * D, B, 256, device="cuda", requires_grad=True)
        c0 = torch.randn(L * D, B, 256, device="cuda", requires_grad=True)
        weights = [w for ws in lstm.all_weights for w in ws]
        seq, (hN, cN), keep = lstm_rec.lstm_stack(x, h0, c0, weights, L, D == 2, dropout=p, return_keep=True)
        assert keep.shape == (L - 1, B, T, D * 256) and keep.dtype == torch.bool
        if p == 1:
            assert not keep.any()
        seq_ref, hN_ref, cN_ref = _oracle(lstm, L, D, p, x, h0, c0, keep)
        torch.testing.assert_close(seq, seq_ref, rtol=3e-3, atol=3e-3)
        torch.testing.assert_close(hN, hN_ref, rtol=3e-3, atol=3e-3)
        torch.testing.assert_close(cN, cN_ref, rtol=3e-3, atol=3e-3)
        g, gh, gc = torch.randn_like(seq), torch.randn_like(hN), torch.randn_like(cN)
        names = ["x", "h0", "c0"] + [n for ns in lstm._all_weights for n in ns]
        ins = [x, h0, c0] + weights
        ref = torch.autograd.grad([seq_ref, hN_ref, cN_ref], ins, [g, gh, gc])
        got = torch.autograd.grad([seq, hN, cN], ins, [g, gh, gc])
        for name, a, b in zip(names, got, ref):
            assert _rel(a, b) < 5e-3, (name, _rel(a, b))
    finally:
        torch.backends.cudnn.allow_tf32 = old


def _stack_inputs(L, D, F, B, T, seed=0):
    torch.manual_seed(seed)
    lstm = torch.nn.LSTM(F, 256, num_layers=L, bidirectional=D == 2, batch_first=True).cuda()
    x = torch.randn(B, T, F, device="cuda")
    h0 = torch.randn(L * D, B, 256, device="cuda")
    c0 = torch.randn(L * D, B, 256, device="cuda")
    return [w.detach() for ws in lstm.all_weights for w in ws], x, h0, c0


@pytest.mark.parametrize("p", [0.1, 0.5])
def test_mask_keep_rate_and_independence(p):
    """The kept fraction of a large mask is within 6 sigma of 1 - p (binomial); masks differ between layers
    and between calls."""
    from distributed_torch_horovod_gcp_b200.ops import lstm_rec
    _kern()
    L, D, F, B, T = 3, 2, 23, 100, 50
    weights, x, h0, c0 = _stack_inputs(L, D, F, B, T)
    with torch.no_grad():
        _, _, k1 = lstm_rec.lstm_stack(x, h0, c0, weights, L, True, dropout=p, return_keep=True)
        _, _, k2 = lstm_rec.lstm_stack(x, h0, c0, weights, L, True, dropout=p, return_keep=True)
    n = k1[0].numel()
    for m in (k1[0], k1[1], k2[0]):
        kept = float(m.float().mean())
        sigma = (p * (1 - p) / n) ** 0.5
        assert abs(kept - (1 - p)) < 6 * sigma, (kept, 1 - p, sigma)
    assert not torch.equal(k1[0], k1[1])
    assert not torch.equal(k1[0], k2[0])
    # independent masks agree on a fraction p^2 + (1 - p)^2 of the elements
    same = float((k1[0] == k2[0]).float().mean())
    assert abs(same - (p * p + (1 - p) ** 2)) < 0.01, same


def test_manual_seed_reproduces_masks_and_outputs():
    from distributed_torch_horovod_gcp_b200.ops import lstm_rec
    _kern()
    L, D, F, B, T = 3, 1, 23, 32, 10
    weights, x, h0, c0 = _stack_inputs(L, D, F, B, T)
    outs = []
    for _ in range(2):
        torch.manual_seed(123)
        with torch.no_grad():
            outs.append(lstm_rec.lstm_stack(x, h0, c0, weights, L, False, dropout=0.4, return_keep=True))
    (s1, (h1, c1), k1), (s2, (h2, c2), k2) = outs
    assert torch.equal(k1, k2)
    assert torch.equal(s1, s2) and torch.equal(h1, h2) and torch.equal(c1, c2)
    with torch.no_grad():
        s3, _ = lstm_rec.lstm_stack(x, h0, c0, weights, L, False, dropout=0.0)
    assert not torch.equal(s1, s3)


def test_dropout_model_runs_without_cudnn(monkeypatch):
    from distributed_torch_horovod_gcp_b200.models import LSTM
    from distributed_torch_horovod_gcp_b200.ops import counters
    _kern()
    torch.manual_seed(0)
    m = LSTM(23, 10, 1, 256, n_layers=2, bidirectional=True, dropout=0.3, device=torch.device("cuda"))

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


def test_eval_mode_matches_no_dropout_model():
    from distributed_torch_horovod_gcp_b200.models import LSTM
    _kern()
    dev = torch.device("cuda")
    torch.manual_seed(0)
    m = LSTM(23, 10, 1, 256, n_layers=3, bidirectional=True, dropout=0.3, device=dev)
    ref = LSTM(23, 10, 1, 256, n_layers=3, bidirectional=True, device=dev)
    ref.load_state_dict(m.state_dict())
    m.eval()
    ref.eval()
    x = torch.randn(32, 10, 23, device=dev)
    with torch.no_grad():
        torch.manual_seed(1)
        out = m(x)
        torch.manual_seed(1)
        out_ref = ref(x)
    assert torch.equal(out, out_ref)


def test_dropout_training_step_and_graph_replay(hvd_single, monkeypatch):
    """A dropout model through hvd.DistributedOptimizer(Adam) with the fused engine: every LSTM gradient goes
    through its grad sink, and a CUDA-graphed step draws a new mask on every replay."""
    monkeypatch.setenv("B200DP_FUSED_SINGLE", "1")
    hvd = hvd_single
    from distributed_torch_horovod_gcp_b200.models import LSTM
    from distributed_torch_horovod_gcp_b200.ops import lstm_rec
    from distributed_torch_horovod_gcp_b200.utils.graph import GraphedStep
    _kern()
    dev = torch.device("cuda", 0)
    torch.manual_seed(0)
    m = LSTM(23, 10, 1, 256, n_layers=2, bidirectional=True, dropout=0.3, device=dev)
    opt = hvd.DistributedOptimizer(torch.optim.Adam(m.parameters(), lr=1e-3), named_parameters=m.named_parameters())
    assert opt.fused_engine is not None
    fired = set()
    for n, p in m.lstm.named_parameters():
        sink = getattr(p, "_b200dp_sink", None)
        assert sink is not None, n

        def rec(f=sink._fire, n=n):
            fired.add(n)
            f()
        sink._fire = rec
    masks = {}
    stack = lstm_rec.lstm_stack

    def spy(*a, **k):                          # keep the mask of the latest forward
        seq, hc, masks["keep"] = stack(*a, return_keep=True, **k)
        return seq, hc
    monkeypatch.setattr(lstm_rec, "lstm_stack", spy)
    B = 32
    x = torch.randn(B, 10, 23, device=dev)
    y = torch.randn(B, 1, 1, device=dev)

    def step(xb, yb):
        loss = torch.nn.functional.mse_loss(m(xb), yb)
        loss.backward()
        opt.step()
        opt.zero_grad()
        return loss.detach()
    l0 = step(x, y)
    torch.cuda.synchronize()
    assert fired == {n for n, _ in m.lstm.named_parameters()}
    assert torch.isfinite(l0)
    graphed = GraphedStep(step, [x, y], warmup=2)
    keeps, losses = [], []
    for _ in range(2):
        losses.append(graphed(x, y).clone())
        keeps.append(masks["keep"].clone())
    torch.cuda.synchronize()
    assert keeps[0].shape == (1, B, 10, 512)
    assert not torch.equal(keeps[0], keeps[1])
    assert all(torch.isfinite(v) for v in losses)


if __name__ == "__main__":
    print(json.dumps({_case_id(c): stack_digests(*c) for c in GOLDEN_CASES}, indent=1))
