"""``ops.functional.lstm`` and ``ops.functional.lstm_head``, the one choice each of the LSTM recurrence's and the
LSTM head's kernel, on both sides of each of their boundaries, alone and through ``models.LSTM``.  No GPU or kernel
library: the library handles are stubs, the device capability is patched, the inputs are CPU tensors that report
themselves as CUDA, and the four paths are recorders."""
import logging

import pytest
import torch
from torch import nn

BF16 = torch.bfloat16


class _OnCuda(torch.Tensor):
    @property
    def is_cuda(self):
        return True


def _cuda(*shape, device="cpu"):
    return torch.zeros(*shape, device=device).as_subclass(_OnCuda)


class _StubLib:
    @staticmethod
    def b200dp_lstm_rec_supported(H, F):
        return 1 if F <= 512 else 0


@pytest.fixture
def calls(monkeypatch):
    """Opens the kernel gate (library loaded, both LSTM ops registered, an sm_90 device) and replaces the four
    paths by recorders; returns the list of the paths taken, in order."""
    from distributed_torch_horovod_gcp_b200.ops import _bind, functional, kernels, lstm_fused, lstm_rec
    lib = _StubLib()
    monkeypatch.setattr(kernels, "_load", lambda: lib)
    monkeypatch.setattr(kernels, "_HAVE", {"lstm_recurrent": True, "lstm_fused": True})
    monkeypatch.setattr(torch.cuda, "get_device_capability", lambda device=None: (9, 0))
    monkeypatch.setattr(lstm_rec, "_lib", lib)
    monkeypatch.setattr(lstm_fused, "_lib", lib)
    monkeypatch.setattr(functional, "_FORCE_REFERENCE", False)
    monkeypatch.delenv("B200DP_DISABLE_KERNELS", raising=False)
    taken = []

    def recurrence(name):
        def run(x, *args, **kwargs):
            taken.append(name)
            B, T = x.shape[:2]
            return _cuda(B, T, 256), (None, None)
        return run

    def head(name):
        def run(seq, t, l1, l2, l3):
            taken.append(name)
            return _cuda(seq.shape[0], 1, l3.out_features)
        return run
    monkeypatch.setattr(lstm_rec, "lstm_stack", recurrence("k5"))
    monkeypatch.setattr(functional, "lstm_reference", recurrence("cudnn"))
    monkeypatch.setattr(_bind, "lstm_head", head("k6"))
    monkeypatch.setattr(functional, "lstm_head_reference", head("torch"))
    return taken


def _lstm(F=23, H=256, dtype=torch.float32, **kw):
    return nn.LSTM(F, H, batch_first=kw.pop("batch_first", True), **kw).to(dtype)


REC_CASES = [   # id, module, input features, expected path
    ("h256", _lstm(), 23, "k5"),
    ("h128", _lstm(H=128), 23, "cudnn"),
    ("bf16-weights", _lstm(dtype=BF16), 23, "cudnn"),
    ("proj-size", _lstm(proj_size=64), 23, "cudnn"),
    ("seq-first", _lstm(batch_first=False), 23, "cudnn"),
    ("2-layer-bidirectional-dropout", _lstm(num_layers=2, bidirectional=True, dropout=0.3), 23, "k5"),
    ("features-512", _lstm(F=512), 512, "k5"),
    ("features-513", _lstm(F=513), 513, "cudnn"),
]


@pytest.mark.parametrize("module,F,expected", [c[1:] for c in REC_CASES], ids=[c[0] for c in REC_CASES])
def test_recurrence(module, F, expected, calls):
    from distributed_torch_horovod_gcp_b200.ops import functional as F2
    F2.lstm(_cuda(4, 10, F), module, (None, None))
    assert calls == [expected]


def test_recurrence_kernel_arguments(calls, monkeypatch):
    """The whole stack's weights in ``nn.LSTM`` order, and inter-layer dropout in training mode only."""
    from distributed_torch_horovod_gcp_b200.ops import functional as F2, lstm_rec
    module = _lstm(num_layers=2, bidirectional=True, dropout=0.3)
    seen = []
    monkeypatch.setattr(lstm_rec, "lstm_stack", lambda *a, **k: seen.append((a, k)) or (None, None))
    x, h0, c0 = _cuda(4, 10, 23), torch.zeros(4, 4, 256), torch.zeros(4, 4, 256)
    for training in (True, False):
        F2.lstm(x, module.train(training), (h0, c0))
    for (args, kwargs), p in zip(seen, (0.3, 0.0)):
        assert args[:3] == (x, h0, c0) and args[4:] == (2, True) and kwargs == {"dropout": p}
        assert len(args[3]) == 16 and all(a is b for a, b in zip(args[3], module.parameters()))


def test_recurrence_logs_cudnn_once_when_the_gate_is_open(calls, monkeypatch, caplog):
    from distributed_torch_horovod_gcp_b200.ops import functional as F2
    monkeypatch.setattr(F2, "_warned_cudnn", False)
    with caplog.at_level(logging.WARNING, logger="b200dp"):
        monkeypatch.setenv("B200DP_DISABLE_KERNELS", "1")
        F2.lstm(_cuda(4, 10, 23), _lstm(H=128), (None, None))
        assert not caplog.records
        monkeypatch.delenv("B200DP_DISABLE_KERNELS")
        for _ in range(2):
            F2.lstm(_cuda(4, 10, 23), _lstm(H=128), (None, None))
    assert calls == ["cudnn"] * 3
    assert len(caplog.records) == 1 and "using the cuDNN RNN" in caplog.records[0].getMessage()


def _head(N1=256, N3=1):
    return nn.Linear(256, N1), nn.Linear(N1, 64), nn.Linear(64, N3)


def _set(linear, name, value):
    with torch.no_grad():
        getattr(linear, name).data = value


HEAD_CASES = [   # id, batch, head, change, expected path
    ("batch-1024", 1024, _head(), None, "k6"),
    ("batch-1025", 1025, _head(), None, "torch"),
    ("sizes-12000", 8, _head(N1=12000 - 256 - 64 - 1), None, "k6"),
    ("sizes-12001", 8, _head(N1=12001 - 256 - 64 - 1), None, "torch"),
    ("linear2-weight-bf16", 8, _head(), lambda h: _set(h[1], "weight", h[1].weight.to(BF16)), "torch"),
    ("linear3-weight-non-contiguous", 8, _head(N3=4),
     lambda h: _set(h[2], "weight", torch.zeros(4, 128)[:, ::2]), "torch"),
    ("linear1-no-bias", 8, (nn.Linear(256, 256, bias=False), nn.Linear(256, 64), nn.Linear(64, 1)), None, "torch"),
]


@pytest.mark.parametrize("B,head,change,expected", [c[1:] for c in HEAD_CASES], ids=[c[0] for c in HEAD_CASES])
def test_head(B, head, change, expected, calls):
    from distributed_torch_horovod_gcp_b200.ops import functional as F2
    if change is not None:
        change(head)
    F2.lstm_head(_cuda(B, 10, 256), 9, *head)
    assert calls == [expected]


@pytest.mark.parametrize("seq,t,expected", [
    (_cuda(8, 10, 256), 0, "k6"),
    (_cuda(8, 10, 256), 10, "torch"),           # past the last step
    (_cuda(8, 10, 128), 9, "torch"),            # seq narrower than linear1's input
    (_cuda(8, 10, 256, device="meta"), 9, "torch"),   # linears on another device than seq
], ids=["t-0", "t-past-end", "seq-width", "other-device"])
def test_head_reads_seq_and_linears_in_bounds(seq, t, expected, calls):
    from distributed_torch_horovod_gcp_b200.ops import functional as F2
    F2.lstm_head(seq, t, *_head())
    assert calls == [expected]


def _set_off(off, monkeypatch):
    from distributed_torch_horovod_gcp_b200.ops import functional, kernels
    if off == "B200DP_DISABLE_KERNELS":
        monkeypatch.setenv(off, "1")
    elif off == "_FORCE_REFERENCE":
        monkeypatch.setattr(functional, off, True)
    elif off == "capability-8.0":
        monkeypatch.setattr(torch.cuda, "get_device_capability", lambda device=None: (8, 0))
    elif off == "library-missing":
        monkeypatch.setattr(kernels, "_load", lambda: None)
    elif off == "ops-not-registered":
        monkeypatch.setattr(kernels, "_HAVE", {})


@pytest.mark.parametrize("off", ["none", "fused=False", "B200DP_DISABLE_KERNELS", "_FORCE_REFERENCE",
                                 "capability-8.0", "library-missing", "ops-not-registered"])
def test_model_takes_both_choices_through_the_gate(off, calls, monkeypatch):
    from distributed_torch_horovod_gcp_b200.models import LSTM
    m = LSTM(23, 10, 1, 256, fused=False if off == "fused=False" else None)
    _set_off(off, monkeypatch)
    out = m(_cuda(32, 10, 23))
    assert out.shape == (32, 1, 1)
    assert calls == (["k5", "k6"] if off == "none" else ["cudnn", "torch"])
