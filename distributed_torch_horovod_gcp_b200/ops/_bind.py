"""ctypes signatures + autograd wrappers for the compute kernels.  ``register`` marks an op
available only if its C symbol exists in the built library."""
from __future__ import annotations

from typing import Dict

from . import gemm as _gemm
from . import bn as _bn
from . import lstm_fused as _lstm
from . import ln as _ln
from . import conv as _conv
from . import lstm_rec as _lstm_rec
from . import attention as _attn
from . import xent as _xent
from . import dropout as _dropout
from .attention import attention_fused  # noqa: F401
from .dropout import dropout_add  # noqa: F401
from .xent import linear_cross_entropy  # noqa: F401
from .lstm_rec import lstm_recurrent  # noqa: F401
from .lstm_fused import head as lstm_head  # noqa: F401
from .conv import conv3x3, conv2d_implicit  # noqa: F401
from .ln import layer_norm  # noqa: F401
from .gemm import linear, mlp, qkv_proj  # noqa: F401  (re-exported as kernels.linear / .mlp / .qkv_proj)
from .bn import conv_bn_act, bn_act, max_pool_3x3_s2, global_avg_pool  # noqa: F401


def register(lib, have: Dict[str, bool]) -> None:
    _gemm.register(lib, have)
    _bn.register(lib, have)
    _lstm.register(lib, have)
    _ln.register(lib, have)
    _conv.register(lib, have)
    _lstm_rec.register(lib, have)
    _attn.register(lib, have)
    _xent.register(lib, have)
    _dropout.register(lib, have)


def linear_supported(x, weight, bias=None, residual=None, w2=None, b2=None) -> bool:
    return _gemm.supported(x, weight, bias, residual, w2, b2)


def layer_norm_supported(x, weight, bias) -> bool:
    return _ln.supported(x, weight, bias)


def linear_cross_entropy_supported(x, weight, targets) -> bool:
    return _xent.supported(x, weight, targets)


def dropout_add_supported(y, residual) -> bool:
    return _dropout.supported(y, residual)


def lstm_head_supported(seq, t_index, l1, l2, l3) -> bool:
    return _lstm.head_supported(seq, t_index, l1, l2, l3)
