"""K5 — persistent LSTM recurrence binding (csrc/lstm_rec_sm90.cu).

``lstm_recurrent(x, h0, c0, w_ih, w_hh, b_ih, b_hh) -> (seq, (hT, cT))`` is a drop-in for a
single-layer unidirectional ``nn.LSTM(batch_first=True)`` call with hidden size 256 (the reference
model, reference app/torch_train.py:121-122,195) in fp32: forward = x-projection kernel + ONE
cluster kernel for all timesteps, backward = ONE cluster kernel + ONE gradient kernel.  Weight
gradients go straight into the gradient-bucket slots when the parameters carry a grad sink
(ops/grad_sink.py).  cuDNN is not involved.
"""
from __future__ import annotations

import ctypes

import torch

from . import counters
from . import grad_sink

_lib = None


def register(lib, have):
    global _lib
    if not hasattr(lib, "b200dp_lstm_rec_fwd"):
        return
    _lib = lib
    vp, i, u64 = ctypes.c_void_p, ctypes.c_int, ctypes.c_uint64
    lib.b200dp_lstm_rec_fwd.argtypes = [vp] * 13 + [i, i, i, u64]
    lib.b200dp_lstm_rec_bwd.argtypes = [vp] * 19 + [i, i, i, u64]
    lib.b200dp_lstm_rec_supported.argtypes = [i, i]
    lib.b200dp_lstm_rec_last_error.restype = ctypes.c_char_p
    have["lstm_recurrent"] = True


def _ck(rc):
    if rc != 0:
        raise RuntimeError("lstm_rec kernels: " + (_lib.b200dp_lstm_rec_last_error() or b"").decode())


def supported(x: torch.Tensor, w_hh: torch.Tensor) -> bool:
    return (_lib is not None and x.is_cuda and x.dtype == torch.float32 and w_hh.dtype == torch.float32
            and x.dim() == 3 and w_hh.shape[1] == 256 and w_hh.shape[0] == 1024
            and bool(_lib.b200dp_lstm_rec_supported(256, x.shape[2])))


def _p(t):
    return t.data_ptr() if t is not None else None


class _LSTMRecFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, h0, c0, w_ih, w_hh, b_ih, b_hh):
        B, T, F = x.shape
        H = w_hh.shape[1]
        dev = x.device
        x = x.contiguous()
        h0 = h0.reshape(B, H).contiguous()
        c0 = c0.reshape(B, H).contiguous()
        need = any(ctx.needs_input_grad)
        seq = torch.empty((B, T, H), dtype=torch.float32, device=dev)
        hT = torch.empty((B, H), dtype=torch.float32, device=dev)
        cT = torch.empty((B, H), dtype=torch.float32, device=dev)
        xp = torch.empty((T, B, 4 * H), dtype=torch.float32, device=dev)
        gates = torch.empty((T, B, 4 * H), dtype=torch.float32, device=dev) if need else None
        cs = torch.empty((T, B, H), dtype=torch.float32, device=dev) if need else None
        st = torch.cuda.current_stream(dev).cuda_stream
        _ck(_lib.b200dp_lstm_rec_fwd(x.data_ptr(), h0.data_ptr(), c0.data_ptr(), w_ih.data_ptr(),
                                     w_hh.data_ptr(), b_ih.data_ptr(), b_hh.data_ptr(), xp.data_ptr(),
                                     seq.data_ptr(), hT.data_ptr(), cT.data_ptr(), _p(gates), _p(cs),
                                     B, T, F, st))
        counters.bump("lstm_rec_fwd", 2)
        if need:
            ctx.save_for_backward(x, h0, c0, w_ih, w_hh, seq, gates, cs)
            ctx.params = (w_ih, w_hh, b_ih, b_hh)
            for prm, ng in zip(ctx.params, ctx.needs_input_grad[3:]):
                if ng:
                    grad_sink.note_forward(prm)
        return seq, hT.view(1, B, H), cT.view(1, B, H)

    @staticmethod
    def backward(ctx, dseq, dhT, dcT):
        x, h0, c0, w_ih, w_hh, seq, gates, cs = ctx.saved_tensors
        B, T, F = x.shape
        H = w_hh.shape[1]
        dev = x.device
        dseq = dseq.contiguous() if dseq is not None else None
        dhT = dhT.reshape(B, H).contiguous() if dhT is not None else None
        dcT = dcT.reshape(B, H).contiguous() if dcT is not None else None
        dG = torch.empty((T, B, 4 * H), dtype=torch.float32, device=dev)
        ni = ctx.needs_input_grad
        dh0 = torch.empty((B, H), dtype=torch.float32, device=dev) if ni[1] else None
        dc0 = torch.empty((B, H), dtype=torch.float32, device=dev) if ni[2] else None
        dx = torch.empty_like(x) if ni[0] else None
        # parameter gradients: into the gradient buckets when possible (first pass of the step only:
        # the kernels overwrite / atomically add onto zero)
        sinks = [grad_sink.begin(prm) for prm in ctx.params]
        direct = all(s[0] is not None and not s[1] for s in sinks) and \
            all(s[0].is_contiguous() for s in sinks)
        if direct:
            dW_ih, dW_hh, db_ih, db_hh = [s[0] for s in sinks]
            dW_hh.zero_()
        else:
            dW_ih = torch.empty_like(w_ih)
            dW_hh = torch.zeros_like(w_hh)
            db_ih = torch.empty(4 * H, dtype=torch.float32, device=dev)
            db_hh = torch.empty(4 * H, dtype=torch.float32, device=dev)
        st = torch.cuda.current_stream(dev).cuda_stream
        _ck(_lib.b200dp_lstm_rec_bwd(x.data_ptr(), h0.data_ptr(), c0.data_ptr(), w_ih.data_ptr(),
                                     w_hh.data_ptr(), seq.data_ptr(), gates.data_ptr(), cs.data_ptr(),
                                     _p(dseq), _p(dhT), _p(dcT), dG.data_ptr(), _p(dh0), _p(dc0),
                                     dW_ih.data_ptr(), dW_hh.data_ptr(), db_ih.data_ptr(), db_hh.data_ptr(),
                                     _p(dx), B, T, F, st))
        counters.bump("lstm_rec_bwd", 2)
        if direct:
            for s in sinks:
                s[2]()
            dW_ih = dW_hh = db_ih = db_hh = None
        return (dx, dh0.view(1, B, H) if dh0 is not None else None,
                dc0.view(1, B, H) if dc0 is not None else None, dW_ih, dW_hh, db_ih, db_hh)


def lstm_recurrent(x, h0, c0, w_ih, w_hh, b_ih, b_hh):
    seq, hT, cT = _LSTMRecFn.apply(x, h0, c0, w_ih, w_hh, b_ih, b_hh)
    return seq, (hT, cT)
