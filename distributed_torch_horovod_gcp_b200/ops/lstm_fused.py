"""K6 — fused linear head of the reference LSTM model (csrc/lstm_kernels.cu): the last-timestep
gather (reference index_select, app/torch_train.py:196) + the three activation-free linears
(app/torch_train.py:199-205) as ONE forward kernel and TWO backward kernels, fp32.  The recurrent
part is the persistent cluster kernel K5 (ops/lstm_rec.py, csrc/lstm_rec_sm90.cu)."""
from __future__ import annotations

import ctypes

import torch

from . import counters

_lib = None


def register(lib, have):
    global _lib
    if not hasattr(lib, "b200dp_head_fwd"):
        return
    _lib = lib
    vp, i, ll, u64 = ctypes.c_void_p, ctypes.c_int, ctypes.c_longlong, ctypes.c_uint64
    lib.b200dp_head_fwd.argtypes = [vp, ll, vp, vp, vp, vp, vp, vp, vp, vp, vp, i, i, i, i, i, u64]
    lib.b200dp_head_bwd.argtypes = [vp, vp, ll, vp, vp, vp, vp, vp, vp, vp, vp, ll, vp, vp, vp, vp, vp, vp,
                                    i, i, i, i, i, u64]
    lib.b200dp_lstm_last_error.restype = ctypes.c_char_p
    have["lstm_fused"] = True


def _ck(rc):
    if rc != 0:
        raise RuntimeError("lstm kernels: " + (_lib.b200dp_lstm_last_error() or b"").decode())


class _HeadFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, seq, t_index, W1, b1, W2, b2, W3, b3):
        B, T, H = seq.shape
        N1, N2, N3 = W1.shape[0], W2.shape[0], W3.shape[0]
        dev = seq.device
        a1 = torch.empty((B, N1), dtype=torch.float32, device=dev)
        a2 = torch.empty((B, N2), dtype=torch.float32, device=dev)
        pred = torch.empty((B, N3), dtype=torch.float32, device=dev)
        x_ptr = seq.data_ptr() + t_index * H * 4
        _ck(_lib.b200dp_head_fwd(x_ptr, T * H, W1.data_ptr(), b1.data_ptr(), W2.data_ptr(), b2.data_ptr(),
                                 W3.data_ptr(), b3.data_ptr(), a1.data_ptr(), a2.data_ptr(),
                                 pred.data_ptr(), B, H, N1, N2, N3,
                                 torch.cuda.current_stream(dev).cuda_stream))
        counters.bump("lstm_head_fwd")
        ctx.save_for_backward(seq, a1, a2, W1, W2, W3)
        ctx.t_index = t_index
        return pred.view(B, 1, N3)

    @staticmethod
    def backward(ctx, dpred):
        seq, a1, a2, W1, W2, W3 = ctx.saved_tensors
        B, T, H = seq.shape
        N1, N2, N3 = W1.shape[0], W2.shape[0], W3.shape[0]
        dev = seq.device
        dp = dpred.reshape(B, N3).contiguous().float()
        da1 = torch.empty_like(a1)
        da2 = torch.empty_like(a2)
        dseq = torch.zeros_like(seq)                    # index_select backward: zeros + last step
        dW1, db1 = torch.empty_like(W1), torch.empty(N1, dtype=torch.float32, device=dev)
        dW2, db2 = torch.empty_like(W2), torch.empty(N2, dtype=torch.float32, device=dev)
        dW3, db3 = torch.empty_like(W3), torch.empty(N3, dtype=torch.float32, device=dev)
        off = ctx.t_index * H * 4
        _ck(_lib.b200dp_head_bwd(dp.data_ptr(), seq.data_ptr() + off, T * H, a1.data_ptr(), a2.data_ptr(),
                                 W1.data_ptr(), W2.data_ptr(), W3.data_ptr(), da1.data_ptr(),
                                 da2.data_ptr(), dseq.data_ptr() + off, T * H, dW1.data_ptr(),
                                 db1.data_ptr(), dW2.data_ptr(), db2.data_ptr(), dW3.data_ptr(),
                                 db3.data_ptr(), B, H, N1, N2, N3,
                                 torch.cuda.current_stream(dev).cuda_stream))
        counters.bump("lstm_head_bwd", 2)
        return dseq, None, dW1, db1, dW2, db2, dW3, db3


def head_supported(seq: torch.Tensor, t_index: int, l1, l2, l3) -> bool:
    """Whether ``l3(l2(l1(seq[:, t_index:t_index + 1])))`` can run on K6: fp32 ``seq`` [B, T, H] with B <= 1024
    and 0 <= ``t_index`` < T, three chained biased linears with H + out1 + out2 + out3 <= 12000, and all six
    of their tensors dense fp32 on ``seq``'s device (the kernels read them by pointer)."""
    tensors = (l1.weight, l1.bias, l2.weight, l2.bias, l3.weight, l3.bias)
    return (_lib is not None and seq.dim() == 3 and seq.dtype == torch.float32 and seq.shape[0] <= 1024
            and 0 <= t_index < seq.shape[1] and l1.in_features == seq.shape[2]
            and l2.in_features == l1.out_features and l3.in_features == l2.out_features
            and l1.in_features + l1.out_features + l2.out_features + l3.out_features <= 12000
            and all(p is not None and p.dtype == torch.float32 and p.is_contiguous() and p.device == seq.device
                    for p in tensors))


def head(seq: torch.Tensor, t_index: int, l1, l2, l3) -> torch.Tensor:
    """``l3(l2(l1(seq[:, t_index:t_index + 1])))`` on K6, ``[B, 1, out3]``; ``head_supported`` must hold."""
    return _HeadFn.apply(seq.contiguous(), t_index, l1.weight, l1.bias, l2.weight, l2.bias, l3.weight, l3.bias)
