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


def available(model, x: torch.Tensor) -> bool:
    if _lib is None:
        try:
            from . import kernels
            kernels.has("lstm_fused")        # triggers the lazy library load + register()
        except Exception:
            return False
    p = model.linear.weight
    return (_lib is not None and x.is_cuda and p.dtype == torch.float32 and x.dtype == torch.float32
            and x.shape[0] <= 1024
            and model.linear.in_features + model.linear.out_features + model.linear2.out_features
            + model.linear3.out_features <= 12000)


_warned_cudnn = False


def forward(model, x, hidden):
    """Persistent recurrence kernel (K5, ops/lstm_rec.py; cuDNN only for shapes it does not cover)
    + fused head (K6)."""
    from . import lstm_rec
    lstm = model.lstm
    if model.n_layers == 1 and lstm_rec.supported(x, lstm.weight_hh_l0):
        seq, model.hidden = lstm_rec.lstm_recurrent(x, hidden[0], hidden[1], lstm.weight_ih_l0,
                                                    lstm.weight_hh_l0, lstm.bias_ih_l0, lstm.bias_hh_l0)
    else:
        global _warned_cudnn
        if not _warned_cudnn:
            _warned_cudnn = True
            import logging
            logging.getLogger("b200dp").warning(
                "LSTM shape (layers=%d, hidden=%d, features=%d, bidirectional=%s) is outside the persistent "
                "recurrence kernel (1 layer, H=256, F<=32): using the cuDNN RNN for this module",
                model.n_layers, model.h_size, model.n_features, model.directions == 2)
        seq, model.hidden = lstm(x, hidden)
    if not seq.is_contiguous():
        seq = seq.contiguous()
    return _HeadFn.apply(seq, model.window_size - 1, model.linear.weight, model.linear.bias,
                         model.linear2.weight, model.linear2.bias, model.linear3.weight,
                         model.linear3.bias)
