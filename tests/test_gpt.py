"""GPT model, token batches and the training script's GPT path on the CPU (reference ops)."""
import os
import re
import subprocess
import sys

import torch

from distributed_torch_horovod_gcp_b200.data import SyntheticTokenBatches
from distributed_torch_horovod_gcp_b200.models import build, gpt_tiny

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_gpt2_parameter_count_and_tied_head():
    m = build("gpt2")
    params = list(m.parameters())
    assert len(params) == 148
    assert sum(p.numel() for p in params) == 124_475_904
    assert m.wte.weight.shape == (50304, 768) and m.wpe.weight.shape == (1024, 768)
    assert build("gpt-tiny").vocab == 512 and build("gpttiny").context == 128


def test_lm_head_is_the_token_embedding():
    """No head parameter of its own: zeroing a row of the token embedding zeroes that logit column."""
    torch.manual_seed(0)
    m = gpt_tiny()
    assert not any(n.startswith(("head", "lm_head")) for n, _ in m.named_parameters())
    idx = torch.randint(0, 512, (2, 16))
    idx[idx == 7] = 8                                  # token 7 is not an input: only the head reads its row
    with torch.no_grad():
        m.wte.weight[7].zero_()
        logits = m(idx)
    assert logits.shape == (32, 512)
    assert torch.equal(logits[:, 7], torch.zeros(32))
    assert bool((logits[:, 8] != 0).all())


def test_gpt_tiny_is_causal_on_the_reference_path():
    torch.manual_seed(1)
    m = gpt_tiny().eval()
    B, S = 2, 100
    idx = torch.randint(0, 512, (B, S))
    with torch.no_grad():
        base = m(idx)
        assert base.shape == (B * S, 512)
        for t in (1, 37, 64, 99):
            alt = idx.clone()
            alt[:, t:] = torch.randint(0, 512, (B, S - t))
            out = m(alt)
            torch.testing.assert_close(out.view(B, S, -1)[:, :t], base.view(B, S, -1)[:, :t], rtol=0, atol=1e-6)
            assert not torch.allclose(out.view(B, S, -1)[:, t:], base.view(B, S, -1)[:, t:])


def test_gpt_rejects_sequences_longer_than_the_context():
    m = gpt_tiny()
    try:
        m(torch.zeros(1, 129, dtype=torch.int64))
    except ValueError as e:
        assert "context" in str(e)
    else:
        raise AssertionError("a 129-token sequence was accepted by a 128-token model")


def test_synthetic_token_batches():
    a = SyntheticTokenBatches(3, 17, 50, "cpu", seed=4)
    b = SyntheticTokenBatches(3, 17, 50, "cpu", seed=4)
    x, y = a.next()
    assert x.shape == (3, 17) and y.shape == (51,)
    assert x.dtype == torch.int64 and y.dtype == torch.int64
    assert int(x.min()) >= 0 and int(x.max()) < 50 and int(y.min()) >= 0 and int(y.max()) < 50
    assert torch.equal(y.view(3, 17)[:, :-1], x[:, 1:])
    x2, y2 = b.next()
    assert torch.equal(x, x2) and torch.equal(y, y2)
    x3, _ = a.next()
    assert not torch.equal(x, x3)


def test_train_script_gpt_tiny_cpu(tmp_path):
    env = dict(os.environ, PYTHONPATH=ROOT, B200DP_OFFLINE="1", OMP_NUM_THREADS="2")
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK"):
        env.pop(k, None)
    r = subprocess.run([sys.executable, os.path.join(ROOT, "app", "torch_train.py"), "--model", "gpt-tiny",
                        "--device", "cpu", "--epochs", "1", "--steps-per-epoch", "2", "--batch-size", "2"],
                       cwd=str(tmp_path), env=env, capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr[-2000:]
    assert re.search(r"epoch: 0, train_loss: [\d.e-]+", r.stdout)
    assert re.search(r"epoch: 0, test_loss: [\d.e-]+", r.stdout)
    assert re.search(r"device: 0, avg_time_per_epoch:[\d.]+", r.stdout)
