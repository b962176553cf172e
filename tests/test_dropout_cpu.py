"""Transformer dropout without a GPU: argument checks, the reference path's semantics, eval-mode identity of
the GPT / ViT models and the entry script's ``--dropout`` flag."""
import importlib.util
import os

import pytest
import torch

from test_app_script import _run

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _f2():
    from distributed_torch_horovod_gcp_b200.ops import functional as F2
    return F2


@pytest.mark.parametrize("p", [-0.1, 1.5, float("nan")])
def test_functional_rejects_p_outside_unit_interval(p):
    F2 = _f2()
    y = torch.zeros(2, 4, 192)
    with pytest.raises(ValueError, match="dropout"):
        F2.dropout_add(y, None, p)
    with pytest.raises(ValueError, match="dropout"):
        F2.attention(y, 3, dropout_p=p)
    with pytest.raises(ValueError, match="dropout"):
        F2.attention_reference(y, 3, dropout_p=p)
    with pytest.raises(ValueError, match="dropout"):
        F2.qkv_attention(torch.zeros(2, 4, 64), torch.zeros(192, 64), torch.zeros(192), 1, dropout_p=p)


@pytest.mark.parametrize("p", [-0.5, 2.0])
def test_attention_fused_and_models_reject_bad_p(p):
    from distributed_torch_horovod_gcp_b200.models import gpt_tiny, vit_tiny
    from distributed_torch_horovod_gcp_b200.models.vit import EncoderBlock
    from distributed_torch_horovod_gcp_b200.ops import attention
    q = torch.zeros(1, 1, 8, 64, dtype=torch.bfloat16)
    with pytest.raises(ValueError, match="dropout"):
        attention.attention_fused(q, q, q, dropout_p=p)
    for make in (lambda: gpt_tiny(dropout=p), lambda: vit_tiny(dropout=p), lambda: vit_tiny(attention_dropout=p),
                 lambda: EncoderBlock(64, 1, 128, dropout=p)):
        with pytest.raises(ValueError, match="dropout"):
            make()


def test_dropout_add_reference_semantics():
    F2 = _f2()
    y, r = torch.randn(64, 32), torch.randn(64, 32)
    torch.manual_seed(5)
    got = F2.dropout_add(y, r, 0.25)
    torch.manual_seed(5)
    assert torch.equal(got, r + torch.nn.functional.dropout(y, 0.25))
    torch.manual_seed(5)
    plain = F2.dropout_add(y, None, 0.25)
    kept = plain != 0
    assert torch.allclose(plain[kept], y[kept] / 0.75)
    assert torch.equal(F2.dropout_add(y, r, 0.0), r + y)
    assert torch.equal(F2.dropout_add(y, None, 0.0), y)
    assert torch.equal(F2.dropout_add(y, r, 1.0), r)


def test_attention_reference_passes_dropout_p():
    F2 = _f2()
    qkv = torch.randn(2, 16, 3 * 128)
    base = F2.attention_reference(qkv, 2)
    assert torch.equal(F2.attention_reference(qkv, 2, dropout_p=0.0), base)
    torch.manual_seed(1)
    a = F2.attention_reference(qkv, 2, causal=True, dropout_p=0.5)
    torch.manual_seed(1)
    b = F2.attention(qkv, 2, causal=True, dropout_p=0.5)
    assert torch.equal(a, b) and not torch.equal(a, F2.attention_reference(qkv, 2, causal=True))
    assert torch.equal(F2.attention_reference(qkv, 2, dropout_p=1.0), torch.zeros_like(base))


@pytest.mark.parametrize("name", ["gpt", "vit"])
def test_eval_mode_matches_model_without_dropout(name):
    from distributed_torch_horovod_gcp_b200.models import gpt_tiny, vit_tiny
    torch.manual_seed(0)
    if name == "gpt":
        ref, drop = gpt_tiny(), gpt_tiny(dropout=0.2)
        x = torch.randint(0, 512, (2, 32))
    else:
        ref, drop = vit_tiny(), vit_tiny(dropout=0.2, attention_dropout=0.3)
        torch.nn.init.normal_(ref.head.weight)         # the head starts at zero, which would hide any difference
        x = torch.randn(2, 3, 32, 32)
    drop.load_state_dict(ref.state_dict())
    ref.eval()
    drop.eval()
    with torch.no_grad():
        assert torch.equal(drop(x), ref(x))
        drop.train()
        torch.manual_seed(3)
        a = drop(x)
        torch.manual_seed(3)
        assert torch.equal(drop(x), a)                 # the reference path draws from torch's generator
        assert not torch.equal(a, ref(x))


def test_models_store_dropout():
    from distributed_torch_horovod_gcp_b200.models import gpt_tiny, vit_tiny
    g = gpt_tiny(dropout=0.1)
    assert g.dropout == 0.1 and all(b.dropout == 0.1 and b.attention_dropout == 0.1 for b in g.layers)
    v = vit_tiny(dropout=0.1, attention_dropout=0.05)
    assert v.dropout == 0.1 and all(b.dropout == 0.1 and b.attention_dropout == 0.05 for b in v.layers)
    assert gpt_tiny().dropout == 0.0 and all(b.dropout == 0.0 for b in vit_tiny().layers)


def _train_module():
    spec = importlib.util.spec_from_file_location("torch_train_for_test", os.path.join(ROOT, "app", "torch_train.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def test_dropout_flag_parsing():
    tt = _train_module()
    a = tt.parse_args(["--model", "gpt-tiny", "--dropout", "0.1"])
    assert a.dropout == 0.1 and tt.dropout_kw(a) == {"dropout": 0.1}
    a = tt.parse_args(["--model", "vit_b_16", "--dropout", "0.1"])
    assert tt.dropout_kw(a) == {"dropout": 0.1, "attention_dropout": 0.1}
    assert tt.parse_args(["--model", "gpt2"]).dropout == 0.0
    assert tt.dropout_kw(tt.parse_args(["--model", "gpt2"])) == {}
    for bad in (["--model", "gpt2", "--dropout", "1.5"], ["--model", "lstm", "--dropout", "0.1"],
                ["--model", "resnet50", "--dropout", "0.1"]):
        with pytest.raises(SystemExit):
            tt.parse_args(bad)


def test_gpt_tiny_cpu_run_with_dropout(tmp_path):
    r = _run(["--device", "cpu", "--model", "gpt-tiny", "--dropout", "0.1", "--batch-size", "2", "--seq-len", "32",
              "--epochs", "1", "--max-steps", "2", "--steps-per-epoch", "2"], cwd=str(tmp_path))
    assert r.returncode == 0, r.stderr[-2000:]
    assert "train_loss" in r.stdout
