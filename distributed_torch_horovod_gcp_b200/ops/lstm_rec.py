"""K5 — persistent LSTM recurrence binding (csrc/lstm_rec_sm90.cu).

``lstm_stack(x, h0, c0, weights, num_layers, bidirectional) -> (seq, (h_n, c_n))`` has the semantics of
``nn.LSTM(batch_first=True)`` with hidden size 256 in fp32, for any number of layers, one or two
directions and 1..512 input features: ``weights`` are the module's parameters in ``nn.LSTM`` order
(``lstm.all_weights`` flattened), ``h0``/``c0`` are ``[layers * directions, B, 256]`` and ``seq`` is
``[B, T, directions * 256]``.  Per layer, forward = x-projection kernel(s) + ONE cluster kernel that runs
both directions as separate clusters of the same launch; backward = ONE cluster kernel + the gradient
kernels, the last of which writes ``dx``, i.e. the ``dseq`` of the layer below.  The directions write their
halves of ``seq`` / ``dseq`` and their slices of ``h_n``/``c_n``/``dh0``/``dc0`` in place.

``lstm_stack(..., dropout=p, training=True)`` is ``nn.LSTM(..., dropout=p)`` in training mode: the output
sequence of every layer but the last is multiplied by ``keep / (1 - p)`` (zero at ``p == 1``) before the next
layer reads it; ``h_n``/``c_n`` and the last layer's output are never dropped.  The keep mask of each dropped
layer is drawn by a Philox4x32-10 kernel from a seed that torch's CUDA generator draws into device memory (so
``torch.manual_seed`` reproduces the masks and a replayed CUDA graph draws fresh ones), stored as one bit per
element of the sequence and read by the next layer's input products: x-projection, ``dW_ih`` and ``dx``.  The
forward recurrence and ``dW_hh`` read the undropped sequence.  ``return_keep=True`` also returns the masks.

``lstm_recurrent(x, h0, c0, w_ih, w_hh, b_ih, b_hh) -> (seq, (hT, cT))`` is the one-layer unidirectional
case (the reference model, reference app/torch_train.py:121-122,195).

Weight gradients go straight into the gradient-bucket slots when the parameters carry a grad sink
(ops/grad_sink.py).  cuDNN is not involved.  Nothing synchronises with the host and every workspace comes
from the caching allocator, so the whole path can be captured in a CUDA graph.
"""
from __future__ import annotations

import ctypes

import torch

from . import counters
from . import grad_sink

_lib = None

H = 256
_SIMT_MAX_F = 32            # inputs up to this width use the register-array x-projection / dW_ih kernels


def register(lib, have):
    global _lib
    if not hasattr(lib, "b200dp_lstm_rec_fwd"):
        return
    _lib = lib
    vp, i, u64 = ctypes.c_void_p, ctypes.c_int, ctypes.c_uint64
    d = ctypes.c_double
    lib.b200dp_lstm_rec_fwd.argtypes = [vp, vp, vp, i, i, i, i, d, vp, vp, vp, u64]
    lib.b200dp_lstm_rec_bwd.argtypes = [vp, vp, vp, vp, vp, i, i, i, i, d, vp, u64]
    lib.b200dp_lstm_rec_supported.argtypes = [i, i]
    lib.b200dp_lstm_rec_last_error.restype = ctypes.c_char_p
    have["lstm_recurrent"] = True


def _ck(rc):
    if rc != 0:
        raise RuntimeError("lstm_rec kernels: " + (_lib.b200dp_lstm_rec_last_error() or b"").decode())


def supported(x: torch.Tensor, w_hh: torch.Tensor) -> bool:
    return (_lib is not None and x.is_cuda and x.dtype == torch.float32 and w_hh.dtype == torch.float32
            and x.dim() == 3 and w_hh.shape[1] == H and w_hh.shape[0] == 4 * H
            and bool(_lib.b200dp_lstm_rec_supported(H, x.shape[2])))


def stack_supported(lstm: torch.nn.LSTM, x: torch.Tensor) -> bool:
    """Whether ``lstm(x, (h0, c0))`` can run on the kernels: hidden size 256, fp32, batch_first, biases,
    1..512 input features, dropout in [0, 1] and no projection."""
    return (isinstance(lstm, torch.nn.LSTM) and lstm.hidden_size == H and lstm.batch_first and lstm.bias
            and 0 <= lstm.dropout <= 1 and getattr(lstm, "proj_size", 0) == 0 and x.dim() == 3
            and x.shape[2] == lstm.input_size and x.shape[0] >= 1 and x.shape[1] >= 1
            and all(p.dtype == torch.float32 for p in lstm.parameters())
            and supported(x, lstm.weight_hh_l0))


def _p(t):
    return t.data_ptr() if t is not None else None


def _ptr_array(tensors):
    return (ctypes.c_void_p * len(tensors))(*[_p(t) for t in tensors])


class _LSTMStackFn(torch.autograd.Function):
    """One node for the whole stack.  ``weights``: 4 tensors (w_ih, w_hh, b_ih, b_hh) per (layer, direction),
    in nn.LSTM order.  ``p``: inter-layer dropout probability (0: none).  The fourth output is the keep-bit
    masks, ``[L - 1, B * T * D * 256 / 32]`` int32 (empty without dropout)."""

    @staticmethod
    def forward(ctx, L, D, p, x, h0, c0, *weights):
        B, T, _ = x.shape
        dev = x.device
        x = x.contiguous()
        h0_shape, c0_shape = h0.shape, c0.shape
        h0 = h0.reshape(L * D, B, H).contiguous()
        c0 = c0.reshape(L * D, B, H).contiguous()
        need = any(ctx.needs_input_grad)
        hN = torch.empty((L * D, B, H), dtype=torch.float32, device=dev)
        cN = torch.empty((L * D, B, H), dtype=torch.float32, device=dev)
        st = torch.cuda.current_stream(dev).cuda_stream
        drop = p > 0 and L > 1
        # one (Philox key, offset) pair per dropped layer, from torch's CUDA generator: no host sync, and a
        # CUDA graph replay draws new ones
        seeds = torch.randint(0, 2 ** 62, (L - 1, 2), dtype=torch.int64, device=dev) if drop else None
        keep = torch.empty((L - 1 if drop else 0, B * T * D * H // 32), dtype=torch.int32, device=dev)
        inp, seqs, gates, cs = x, [], [], []
        for l in range(L):
            F = inp.shape[2]
            seq = torch.empty((B, T, D * H), dtype=torch.float32, device=dev)
            ptrs, g_l, c_l = [], [], []
            for d in range(D):
                i = l * D + d
                w_ih, w_hh, b_ih, b_hh = weights[4 * i:4 * i + 4]
                xp = torch.empty((T, B, 4 * H), dtype=torch.float32, device=dev)
                g = torch.empty((T, B, 4 * H), dtype=torch.float32, device=dev) if need else None
                c = torch.empty((T, B, H), dtype=torch.float32, device=dev) if need else None
                g_l.append(g)
                c_l.append(c)
                # per-direction pointer group, in the order of the FW_* enum of csrc/lstm_rec_sm90.cu
                ptrs += [w_ih, w_hh, b_ih, b_hh, h0[i], c0[i], xp, g, c, hN[i], cN[i]]
            keep_in = keep[l - 1] if drop and l > 0 else None
            keep_out = keep[l] if drop and l < L - 1 else None
            _ck(_lib.b200dp_lstm_rec_fwd(inp.data_ptr(), seq.data_ptr(), _ptr_array(ptrs), D, B, T, F, p,
                                         _p(keep_in), _p(seeds[l] if keep_out is not None else None),
                                         _p(keep_out), st))
            counters.bump("lstm_rec_fwd", (D if F <= _SIMT_MAX_F else 1) + 1 + (keep_out is not None))
            seqs.append(seq)
            gates.append(g_l)
            cs.append(c_l)
            inp = seq
        ctx.mark_non_differentiable(keep)
        if need:
            ctx.save_for_backward(x, h0, c0, keep, *seqs, *[t for g_l in gates for t in g_l],
                                  *[t for c_l in cs for t in c_l], *weights)
            ctx.L, ctx.D, ctx.p, ctx.h0_shape, ctx.c0_shape = L, D, p, h0_shape, c0_shape
            for prm, ng in zip(weights, ctx.needs_input_grad[6:]):
                if ng:
                    grad_sink.note_forward(prm)
        return seqs[-1], hN, cN, keep

    @staticmethod
    def backward(ctx, dseq, dhN, dcN, _dkeep):
        L, D, p = ctx.L, ctx.D, ctx.p
        saved = ctx.saved_tensors
        x, h0, c0, keep = saved[:4]
        seqs = saved[4:4 + L]
        gates = saved[4 + L:4 + L + L * D]
        cs = saved[4 + L + L * D:4 + L + 2 * L * D]
        weights = saved[4 + L + 2 * L * D:]
        B, T, _ = x.shape
        dev = x.device
        ni = ctx.needs_input_grad
        dcur = dseq.contiguous() if dseq is not None else None
        dhN = dhN.contiguous() if dhN is not None else None
        dcN = dcN.contiguous() if dcN is not None else None
        dh0 = torch.empty((L * D, B, H), dtype=torch.float32, device=dev) if ni[4] else None
        dc0 = torch.empty((L * D, B, H), dtype=torch.float32, device=dev) if ni[5] else None
        grads = [None] * len(weights)
        st = torch.cuda.current_stream(dev).cuda_stream
        for l in reversed(range(L)):
            inp = x if l == 0 else seqs[l - 1]
            F = inp.shape[2]
            # dx of a layer above the first is the gradient of the layer below's undropped output
            keep_in = keep[l - 1] if keep.shape[0] and l > 0 else None
            dx = torch.empty_like(inp) if (l > 0 or ni[3]) else None
            ptrs, fire = [], []
            for d in range(D):
                i = l * D + d
                prm = weights[4 * i:4 * i + 4]
                # parameter gradients: into the gradient buckets when possible (first pass of the step only:
                # the kernels overwrite / atomically add onto zero)
                sinks = [grad_sink.begin(p) for p in prm]
                if all(s[0] is not None and not s[1] and s[0].is_contiguous() for s in sinks):
                    dW_ih, dW_hh, db_ih, db_hh = [s[0] for s in sinks]
                    dW_hh.zero_()
                    fire += [s[2] for s in sinks]
                else:
                    dW_ih = torch.empty_like(prm[0])
                    dW_hh = torch.zeros_like(prm[1])
                    db_ih = torch.empty(4 * H, dtype=torch.float32, device=dev)
                    db_hh = torch.empty(4 * H, dtype=torch.float32, device=dev)
                    grads[4 * i:4 * i + 4] = [dW_ih, dW_hh, db_ih, db_hh]
                dG = torch.empty((T, B, 4 * H), dtype=torch.float32, device=dev)
                # per-direction pointer group, in the order of the BW_* enum of csrc/lstm_rec_sm90.cu
                ptrs += [prm[0], prm[1], h0[i], c0[i], gates[i], cs[i],
                         dhN[i] if dhN is not None else None, dcN[i] if dcN is not None else None, dG,
                         dh0[i] if dh0 is not None else None, dc0[i] if dc0 is not None else None,
                         dW_ih, dW_hh, db_ih, db_hh]
            _ck(_lib.b200dp_lstm_rec_bwd(inp.data_ptr(), seqs[l].data_ptr(), _p(dcur), _p(dx), _ptr_array(ptrs),
                                         D, B, T, F, p, _p(keep_in), st))
            simt = F <= _SIMT_MAX_F
            counters.bump("lstm_rec_bwd", 1 + D + (0 if simt else 2) + (1 if dx is not None and not (simt and D == 1)
                                                                        else 0))
            for f in fire:
                f()
            dcur = dx
        return (None, None, None, dcur if ni[3] else None,
                dh0.view(ctx.h0_shape) if dh0 is not None else None,
                dc0.view(ctx.c0_shape) if dc0 is not None else None, *grads)


def lstm_stack(x, h0, c0, weights, num_layers: int, bidirectional: bool, dropout: float = 0.0,
               training: bool = True, return_keep: bool = False):
    """``nn.LSTM(batch_first=True, dropout=dropout)`` forward on the K5 kernels (see the module docstring).
    Dropout applies when ``training`` and ``num_layers > 1``.  With ``return_keep`` the result is
    ``seq, (h_n, c_n), keep``: ``keep[l]`` is the bool mask ``[B, T, directions * 256]`` applied to layer
    ``l``'s output (``num_layers - 1`` masks; none without dropout)."""
    D = 2 if bidirectional else 1
    weights = list(weights)
    if len(weights) != 4 * num_layers * D:
        raise ValueError(f"expected {4 * num_layers * D} weight tensors (w_ih, w_hh, b_ih, b_hh per layer and "
                         f"direction), got {len(weights)}")
    if not 0 <= dropout <= 1:
        raise ValueError(f"dropout must be in [0, 1], got {dropout}")
    p = float(dropout) if training else 0.0
    seq, hN, cN, keep = _LSTMStackFn.apply(num_layers, D, p, x, h0, c0, *weights)
    if not return_keep:
        return seq, (hN, cN)
    B, T = x.shape[0], x.shape[1]
    bits = keep.unsqueeze(-1) >> torch.arange(32, dtype=torch.int32, device=keep.device)
    return seq, (hN, cN), (bits & 1).bool().reshape(keep.shape[0], B, T, D * H)


def lstm_recurrent(x, h0, c0, w_ih, w_hh, b_ih, b_hh):
    seq, hT, cT, _ = _LSTMStackFn.apply(1, 1, 0.0, x, h0, c0, w_ih, w_hh, b_ih, b_hh)
    return seq, (hT, cT)
