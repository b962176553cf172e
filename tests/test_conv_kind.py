"""``ops.conv.kind``, the one choice of a convolution's kernel, on both sides of each of its boundaries.  No GPU or
kernel library: the library handles are stubs and the activation is a CPU tensor that reports itself as CUDA."""
import pytest
import torch
from torch import nn

BF16 = torch.bfloat16


class _OnCuda(torch.Tensor):
    @property
    def is_cuda(self):
        return True


def _x(N, C, H, W, grad=False, cl=True, dtype=BF16, cuda=True):
    x = torch.zeros(N, C, H, W, dtype=dtype)
    x = x.contiguous(memory_format=torch.channels_last) if cl else x
    x = x.as_subclass(_OnCuda) if cuda else x
    return x.requires_grad_(grad)


def _conv(cin, cout, k, stride=1, pad=None, bias=False):
    return nn.Conv2d(cin, cout, k, stride, (k - 1) // 2 if pad is None else pad, bias=bias).to(BF16)


@pytest.fixture
def conv_mod(monkeypatch):
    from distributed_torch_horovod_gcp_b200.ops import bn, conv, gemm
    lib = type("StubLib", (), {"b200dp_stem_im2col": None})()
    for mod in (bn, conv, gemm):
        monkeypatch.setattr(mod, "_lib", lib)
    return conv


CASES = [   # id, x, conv, expected kind
    ("1x1-s1", _x(2, 16, 5, 7), _conv(16, 32, 1), "gemm"),
    ("1x1-s2", _x(2, 16, 6, 8), _conv(16, 32, 1, 2), "implicit"),
    ("1x1-s2-odd-H", _x(2, 16, 7, 8), _conv(16, 32, 1, 2), None),
    ("1x1-s1-cin8", _x(2, 8, 5, 7), _conv(8, 32, 1), "gemm"),
    ("1x1-s1-cout12", _x(2, 16, 5, 7), _conv(16, 12, 1), None),
    ("1x1-s1-bias", _x(2, 16, 5, 7), _conv(16, 32, 1, bias=True), None),
    ("stem", _x(2, 3, 32, 64), _conv(3, 64, 7, 2), "stem"),
    ("stem-x-requires-grad", _x(2, 3, 32, 64, grad=True), _conv(3, 64, 7, 2), None),
    ("stem-W-not-multiple-of-8", _x(2, 3, 32, 60), _conv(3, 64, 7, 2), None),
    ("stem-bias", _x(2, 3, 32, 64), _conv(3, 64, 7, 2, bias=True), None),
    ("3x3-s1-cin16", _x(2, 16, 5, 7), _conv(16, 32, 3), "implicit"),
    ("3x3-s1-cin8", _x(2, 8, 5, 7), _conv(8, 32, 3), None),
    ("3x3-s2", _x(2, 16, 6, 8), _conv(16, 32, 3, 2), "implicit"),
    ("3x3-s2-odd-H", _x(2, 16, 7, 8), _conv(16, 32, 3, 2), None),
    ("3x3-pad0", _x(2, 16, 6, 8), _conv(16, 32, 3, pad=0), None),
    ("3x3-padding-same", _x(2, 16, 6, 8), _conv(16, 32, 3, pad="same"), None),
    ("3x3-bias", _x(2, 16, 6, 8), _conv(16, 32, 3, bias=True), None),
    ("x-nchw", _x(2, 16, 5, 7, cl=False), _conv(16, 32, 1), None),
    ("x-fp32", _x(2, 16, 5, 7, dtype=torch.float32), _conv(16, 32, 1), None),
    ("x-on-cpu", _x(2, 16, 5, 7, cuda=False), _conv(16, 32, 1), None),
]


@pytest.mark.parametrize("x,conv,expected", [c[1:] for c in CASES], ids=[c[0] for c in CASES])
def test_kind(x, conv, expected, conv_mod):
    assert conv_mod.kind(x, conv) == expected


# switch or library turned off, case, kind without it
OFF_CASES = [
    ("_USE_GEMM_1X1", "1x1-s1", "implicit"),
    ("_USE_GEMM_1X1", "1x1-s1-cin8", None),
    ("_USE_STEM_GEMM", "stem", None),
    ("_ENABLED", "3x3-s1-cin16", None),
    ("_ENABLED", "1x1-s2", None),
    ("gemm._lib", "1x1-s1", "implicit"),
    ("gemm._lib", "stem", None),
    ("bn._lib", "stem", None),
    ("conv._lib", "3x3-s2", None),
]


@pytest.mark.parametrize("off,case,expected", OFF_CASES, ids=[f"{o}-{c}" for o, c, _ in OFF_CASES])
def test_kind_switched_off(off, case, expected, conv_mod, monkeypatch):
    from distributed_torch_horovod_gcp_b200.ops import bn, gemm
    x, conv, on = next(c[1:] for c in CASES if c[0] == case)
    assert conv_mod.kind(x, conv) == on != expected
    if off.endswith("._lib"):
        monkeypatch.setattr({"bn": bn, "gemm": gemm, "conv": conv_mod}[off.split(".")[0]], "_lib", None)
    else:
        monkeypatch.setattr(conv_mod, off, False)
    assert conv_mod.kind(x, conv) == expected
