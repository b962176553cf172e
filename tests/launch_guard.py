"""A host-side guard for the kernel launches of the ctypes bindings: before a ``b200dp_*`` entry point runs, every
device pointer it is given must be aligned as the kernels load it, and the bytes the kernels read or write through
it must lie inside ONE live block of torch's caching allocator.  A call that fails raises ``GuardError`` and never
reaches the library, so a test can feed an op inputs a predicate might wrongly accept without a kernel ever
touching memory it does not own.

``TABLE`` lists, per entry point, its arguments in the order of the C signature and, for each pointer argument,
the byte extent as a formula of the call's scalar arguments, the alignment and whether it may be null.  The
extents and alignments come from the kernels in ``csrc/``:
- GEMM (gemm_sm90.cu, sm90_common.cuh): A / B / C through TMA descriptors (16-byte base); the residual is read
  in 16-byte vectors (``res_load``), the pre-activation stored in bf16 pairs (4 bytes), bias elements one by one;
  the [M, ldc] matrices span (M - 1) ldc + N elements.
- BatchNorm, pooling, LayerNorm, dropout (elementwise.cu): activations in uint4 vectors, parameters through
  ``ld_param`` / ``st_param`` one element at a time in the dtype ``param_bf16`` names, max-pool indices as uint2.
- convolution (conv_sm90.cu): NHWC / KRSC tensors through TMA; OH = (H + 2 pad - R) / stride + 1.
- attention (attn_sm90.cu): [B, H, S, D] tensors with element strides from the host arrays, 16-byte rows.
- LM-head cross-entropy (xent_sm90.cu): x and W through TMA, int64 targets, fp32 row vectors.
Entry points of the library that launch nothing (``*_supported``, ``*_last_error``) pass through; any other
``b200dp_*`` symbol raises, so a new entry point cannot run unguarded."""
from __future__ import annotations

import bisect
import ctypes
from collections import Counter


class GuardError(Exception):
    """A launch whose pointer arguments the kernels would misuse (not a RuntimeError, so a test that expects the
    reference path's RuntimeError does not take it for one)."""


def _p(a):
    """Bytes per BN / LayerNorm parameter element: ``param_bf16`` selects bf16, else fp32."""
    return 2 if a.param_bf16 else 4


def _mat(rows, ld, cols):
    """Elements spanned by a [rows, cols] matrix with leading dimension ld (0 for no rows)."""
    return (rows - 1) * ld + cols if rows > 0 and cols > 0 else 0


def _span4(a, st, D):
    """Elements spanned by a [B, H, S, D] tensor with (batch, head, seq) element strides st (a ctypes array)."""
    if a.B <= 0 or a.H <= 0 or a.S <= 0:
        return 0
    return (a.B - 1) * st[0] + (a.H - 1) * st[1] + (a.S - 1) * st[2] + D


def _pool_out(n):
    return (n - 1) // 2 + 1


def _conv_out(a, n):
    return (n + 2 * a.pad - a.R) // a.stride + 1


# pointer spec: name -> (extent in bytes as a function of the scalar arguments, alignment, required)
# required may be a function of the arguments (e.g. the ReLU mask only with relu != 0)
REQ, OPT = True, False
_GEMM_ARGS = ("A", "B", "C", "M", "N", "K", "lda", "ldb", "ldc", "a_mn", "b_mn", "bias_bf16", "bias_f32",
              "residual", "preact", "act", "out_mode", "out_bf16", "alpha", "splits", "block_n", "max_ctas", "stats",
              "res_mask", "stream")
_ATTN_FWD = ("q", "k", "v", "o", "lse", "B", "H", "S", "D", "sq", "sk", "sv", "so", "scale")
_ATTN_BWD = ("q", "k", "v", "o", "do", "lse", "delta", "acc", "dk", "dv", "B", "H", "S", "D", "sq", "sk", "sv", "so",
             "sdo", "sacc", "sdk", "sdv", "scale", "causal")


def _attn_fwd_ptrs():
    return {"q": (lambda a: 2 * _span4(a, a.sq, a.D), 16, REQ), "k": (lambda a: 2 * _span4(a, a.sk, a.D), 16, REQ),
            "v": (lambda a: 2 * _span4(a, a.sv, a.D), 16, REQ), "o": (lambda a: 2 * _span4(a, a.so, a.D), 16, REQ),
            "lse": (lambda a: 4 * a.B * a.H * a.S, 4, OPT)}


def _attn_bwd_ptrs():
    d = {n: (lambda a, s="s" + n: 2 * _span4(a, getattr(a, s), a.D), 16, REQ)
         for n in ("q", "k", "v", "o", "do", "dk", "dv")}
    d["acc"] = (lambda a: 4 * _span4(a, a.sacc, a.D), 16, REQ)
    d["lse"] = (lambda a: 4 * a.B * a.H * a.S, 4, REQ)
    d["delta"] = (lambda a: 4 * a.B * a.H * a.S, 4, REQ)
    return d


TABLE = {
    "b200dp_gemm_bf16": (_GEMM_ARGS, {
        "A": (lambda a: 2 * (_mat(a.K, a.lda, a.M) if a.a_mn else _mat(a.M, a.lda, a.K)), 16, REQ),
        "B": (lambda a: 2 * (_mat(a.K, a.ldb, a.N) if a.b_mn else _mat(a.N, a.ldb, a.K)), 16, REQ),
        "C": (lambda a: (2 if (a.out_mode == 0 or a.out_bf16) else 4) * _mat(a.M, a.ldc, a.N), 16, REQ),
        "bias_bf16": (lambda a: 2 * a.N, 2, OPT),
        "bias_f32": (lambda a: 4 * a.N, 4, OPT),
        "residual": (lambda a: 2 * _mat(a.M, a.ldc, a.N), 16, OPT),
        "preact": (lambda a: 2 * _mat(a.M, a.ldc, a.N), 4, OPT),
        "stats": (lambda a: 8 * a.N, 4, OPT),
        "res_mask": (lambda a: a.M * (a.N // 8), 1, OPT),
    }),
    "b200dp_bn_fwd": (("x", "res", "y", "gamma", "beta", "stats", "mean", "invstd", "a", "b", "running_mean",
                       "running_var", "M", "C", "eps", "momentum", "relu", "param_bf16", "have_stats", "relu_mask",
                       "nbt", "stream"), {
        "x": (lambda a: 2 * a.M * a.C, 16, REQ), "res": (lambda a: 2 * a.M * a.C, 16, OPT),
        "y": (lambda a: 2 * a.M * a.C, 16, REQ),
        "gamma": (lambda a: _p(a) * a.C, 2, OPT), "beta": (lambda a: _p(a) * a.C, 2, OPT),
        "stats": (lambda a: 8 * a.C, 4, REQ), "mean": (lambda a: 4 * a.C, 4, REQ),
        "invstd": (lambda a: 4 * a.C, 4, REQ), "a": (lambda a: 4 * a.C, 4, REQ), "b": (lambda a: 4 * a.C, 4, REQ),
        "running_mean": (lambda a: _p(a) * a.C, 2, OPT), "running_var": (lambda a: _p(a) * a.C, 2, OPT),
        "relu_mask": (lambda a: a.M * (a.C // 8), 1, lambda a: bool(a.relu)),
        "nbt": (lambda a: 8, 8, OPT),
    }),
    "b200dp_bn_apply": (("x", "res", "y", "a", "b", "M", "C", "relu", "stream"), {
        "x": (lambda a: 2 * a.M * a.C, 16, REQ), "res": (lambda a: 2 * a.M * a.C, 16, OPT),
        "y": (lambda a: 2 * a.M * a.C, 16, REQ), "a": (lambda a: 4 * a.C, 4, REQ), "b": (lambda a: 4 * a.C, 4, REQ),
    }),
    "b200dp_bn_bwd": (("dy", "x", "relu_mask", "dx", "dres", "scale_a", "mean", "invstd", "sums", "dgamma", "dbeta",
                       "param_bf16", "M", "C", "relu", "stream"), {
        "dy": (lambda a: 2 * a.M * a.C, 16, REQ), "x": (lambda a: 2 * a.M * a.C, 16, REQ),
        "relu_mask": (lambda a: a.M * (a.C // 8), 1, lambda a: bool(a.relu)),
        "dx": (lambda a: 2 * a.M * a.C, 16, REQ), "dres": (lambda a: 2 * a.M * a.C, 16, OPT),
        "scale_a": (lambda a: 4 * a.C, 4, REQ), "mean": (lambda a: 4 * a.C, 4, REQ),
        "invstd": (lambda a: 4 * a.C, 4, REQ), "sums": (lambda a: 8 * a.C, 4, REQ),
        "dgamma": (lambda a: _p(a) * a.C, 2, OPT), "dbeta": (lambda a: _p(a) * a.C, 2, OPT),
    }),
    "b200dp_maxpool_fwd": (("x", "y", "idx", "N", "H", "W", "C", "stream"), {
        "x": (lambda a: 2 * a.N * a.H * a.W * a.C, 16, REQ),
        "y": (lambda a: 2 * a.N * _pool_out(a.H) * _pool_out(a.W) * a.C, 16, REQ),
        "idx": (lambda a: a.N * _pool_out(a.H) * _pool_out(a.W) * a.C, 8, REQ),
    }),
    "b200dp_maxpool_bwd": (("dy", "idx", "dx", "N", "H", "W", "C", "stream"), {
        "dy": (lambda a: 2 * a.N * _pool_out(a.H) * _pool_out(a.W) * a.C, 16, REQ),
        "idx": (lambda a: a.N * _pool_out(a.H) * _pool_out(a.W) * a.C, 8, REQ),
        "dx": (lambda a: 2 * a.N * a.H * a.W * a.C, 16, REQ),
    }),
    "b200dp_avgpool_fwd": (("x", "y", "N", "HW", "C", "stream"), {
        "x": (lambda a: 2 * a.N * a.HW * a.C, 16, REQ), "y": (lambda a: 2 * a.N * a.C, 16, REQ),
    }),
    "b200dp_avgpool_bwd": (("dy", "dx", "N", "HW", "C", "stream"), {
        "dy": (lambda a: 2 * a.N * a.C, 16, REQ), "dx": (lambda a: 2 * a.N * a.HW * a.C, 16, REQ),
    }),
    "b200dp_stem_im2col": (("x", "out", "N", "H", "W", "stream"), {
        "x": (lambda a: 2 * a.N * a.H * a.W * 3, 2, REQ),
        "out": (lambda a: 2 * a.N * (a.H // 2) * (a.W // 2) * 168, 16, REQ),
    }),
    "b200dp_ln_fwd": (("x", "y", "gamma", "beta", "mean", "rstd", "rows", "C", "eps", "param_bf16", "stream"), {
        "x": (lambda a: 2 * a.rows * a.C, 16, REQ), "y": (lambda a: 2 * a.rows * a.C, 16, REQ),
        "gamma": (lambda a: _p(a) * a.C, 2, REQ), "beta": (lambda a: _p(a) * a.C, 2, REQ),
        "mean": (lambda a: 4 * a.rows, 4, REQ), "rstd": (lambda a: 4 * a.rows, 4, REQ),
    }),
    "b200dp_ln_bwd": (("dy", "x", "dx", "gamma", "mean", "rstd", "sums", "dgamma", "dbeta", "rows", "C", "param_bf16",
                       "stream"), {
        "dy": (lambda a: 2 * a.rows * a.C, 16, REQ), "x": (lambda a: 2 * a.rows * a.C, 16, REQ),
        "dx": (lambda a: 2 * a.rows * a.C, 16, REQ), "gamma": (lambda a: _p(a) * a.C, 2, REQ),
        "mean": (lambda a: 4 * a.rows, 4, REQ), "rstd": (lambda a: 4 * a.rows, 4, REQ),
        "sums": (lambda a: 8 * a.C, 4, REQ),
        "dgamma": (lambda a: _p(a) * a.C, 2, REQ), "dbeta": (lambda a: _p(a) * a.C, 2, REQ),
    }),
    "b200dp_conv_fprop": (("x", "w", "y", "N", "H", "W", "Cin", "Cout", "R", "S", "stride", "pad", "block_n",
                           "max_ctas", "stats", "stream"), {
        "x": (lambda a: 2 * a.N * a.H * a.W * a.Cin, 16, REQ), "w": (lambda a: 2 * a.Cout * a.R * a.S * a.Cin, 16, REQ),
        "y": (lambda a: 2 * a.N * _conv_out(a, a.H) * _conv_out(a, a.W) * a.Cout, 16, REQ),
        "stats": (lambda a: 8 * a.Cout, 4, OPT),
    }),
    "b200dp_conv_dgrad": (("dy", "w", "dx", "N", "H", "W", "Cin", "Cout", "R", "S", "stride", "pad", "block_n",
                           "max_ctas", "stream"), {
        "dy": (lambda a: 2 * a.N * _conv_out(a, a.H) * _conv_out(a, a.W) * a.Cout, 16, REQ),
        "w": (lambda a: 2 * a.Cout * a.R * a.S * a.Cin, 16, REQ), "dx": (lambda a: 2 * a.N * a.H * a.W * a.Cin, 16, REQ),
    }),
    "b200dp_conv_wgrad": (("dy", "x", "dw", "N", "H", "W", "Cin", "Cout", "R", "S", "stride", "pad", "splits",
                           "block_n", "max_ctas", "accumulate", "out_bf16", "stream"), {
        "dy": (lambda a: 2 * a.N * _conv_out(a, a.H) * _conv_out(a, a.W) * a.Cout, 16, REQ),
        "x": (lambda a: 2 * a.N * a.H * a.W * a.Cin, 16, REQ),
        "dw": (lambda a: (2 if a.out_bf16 else 4) * a.Cout * a.R * a.S * a.Cin, 16, REQ),
    }),
    "b200dp_attn_fwd": (_ATTN_FWD + ("stream",), _attn_fwd_ptrs()),
    "b200dp_attn_fwd_ex": (_ATTN_FWD + ("causal", "stream"), _attn_fwd_ptrs()),
    "b200dp_attn_fwd_dropout": (_ATTN_FWD + ("causal", "seed", "p", "stream"),
                                {**_attn_fwd_ptrs(), "seed": (lambda a: 16, 8, REQ)}),
    "b200dp_attn_bwd": (_ATTN_BWD + ("stream",), _attn_bwd_ptrs()),
    "b200dp_attn_bwd_dropout": (_ATTN_BWD + ("seed", "p", "stream"),
                                {**_attn_bwd_ptrs(), "seed": (lambda a: 16, 8, REQ)}),
    "b200dp_cast_acc_zero": (("src", "dst", "n", "out_bf16", "accumulate", "zero_src", "stream"), {
        "src": (lambda a: 4 * a.n, 16, REQ),
        "dst": (lambda a: (2 if a.out_bf16 else 4) * a.n, lambda a: 8 if a.out_bf16 else 16, REQ),
    }),
    "b200dp_dropout_add": (("y", "res", "out", "n", "seed", "p", "stream"), {
        "y": (lambda a: 2 * a.n, 16, REQ), "res": (lambda a: 2 * a.n, 16, OPT), "out": (lambda a: 2 * a.n, 16, REQ),
        "seed": (lambda a: 16, 8, REQ),
    }),
    "b200dp_xent_fwd": (("x", "w", "t", "lse", "rows", "stats", "out", "N", "D", "V", "ignore_index", "mean",
                         "max_ctas", "stream"), {
        "x": (lambda a: 2 * a.N * a.D, 16, REQ), "w": (lambda a: 2 * a.V * a.D, 16, REQ),
        "t": (lambda a: 8 * a.N, 8, REQ), "lse": (lambda a: 4 * a.N, 4, REQ), "rows": (lambda a: 4 * a.N, 4, OPT),
        "stats": (lambda a: 8, 4, OPT), "out": (lambda a: 4, 4, OPT),
    }),
    "b200dp_xent_grad": (("x", "w", "t", "lse", "g", "per_row", "count", "dl", "c0", "rows", "N", "D", "V",
                          "ignore_index", "max_ctas", "stream"), {
        "x": (lambda a: 2 * a.N * a.D, 16, REQ), "w": (lambda a: 2 * a.V * a.D, 16, REQ),
        "t": (lambda a: 8 * a.N, 8, REQ), "lse": (lambda a: 4 * a.N, 4, REQ),
        "g": (lambda a: 4 * (a.N if a.per_row else 1), 4, REQ), "count": (lambda a: 4, 4, OPT),
        "dl": (lambda a: 2 * a.rows * a.V, 16, REQ),
    }),
}
PASS_THROUGH = ("b200dp_bn_supported", "b200dp_ln_supported")


class _Args:
    def __init__(self, names, values):
        if len(names) != len(values):
            raise GuardError(f"expected {len(names)} arguments, got {len(values)}")
        self.__dict__.update(zip(names, values))


def _ptr(v):
    if v is None:
        return 0
    if isinstance(v, ctypes.c_void_p):
        return v.value or 0
    return int(v)


def live_blocks():
    """[(start, end)] of every live block of torch's caching allocator (requested bytes, not the rounded size)."""
    import torch
    out = []
    for seg in torch.cuda.memory_snapshot():
        addr = seg["address"]
        for b in seg["blocks"]:
            start = b.get("address", addr)
            if b["state"] == "active_allocated":
                out.append((start, start + b.get("requested_size", b["size"])))
            addr = start + b["size"]
    return sorted(out)


def check(symbol, values, blocks):
    """Raise GuardError unless every pointer argument of ``symbol`` called with ``values`` is aligned and its
    extent lies inside one of ``blocks`` (sorted (start, end) pairs)."""
    if symbol not in TABLE:
        raise GuardError(f"{symbol}: no entry in the launch table")
    names, ptrs = TABLE[symbol]
    a = _Args(names, values)
    starts = [b[0] for b in blocks]
    for name, (extent, align, required) in ptrs.items():
        p = _ptr(getattr(a, name))
        req = required(a) if callable(required) else required
        if p == 0:
            if req:
                raise GuardError(f"{symbol}: {name} is null")
            continue
        al = align(a) if callable(align) else align
        if p % al:
            raise GuardError(f"{symbol}: {name} = {p:#x} is not {al}-byte aligned")
        n = extent(a)
        if n < 0:
            raise GuardError(f"{symbol}: {name} has a negative extent {n}")
        i = bisect.bisect_right(starts, p) - 1
        if i < 0 or p > blocks[i][1] or (p == blocks[i][1] and n > 0):
            raise GuardError(f"{symbol}: {name} = {p:#x} points into no live allocation")
        if p + n > blocks[i][1]:
            nxt = i + 1 < len(blocks) and blocks[i + 1][0] < p + n
            what = "spans two allocations" if nxt else "runs past the end of its allocation"
            raise GuardError(f"{symbol}: {name} [{p:#x}, +{n}) {what} [{blocks[i][0]:#x}, {blocks[i][1]:#x})")


class GuardedLib:
    """Stands in for the ctypes library object of the bindings: table entry points are checked against the live
    allocations and counted in ``calls`` before they are forwarded."""

    def __init__(self, lib, calls: Counter, blocks=live_blocks):
        object.__setattr__(self, "_lib", lib)
        object.__setattr__(self, "_calls", calls)
        object.__setattr__(self, "_blocks", blocks)

    def __getattr__(self, name):
        fn = getattr(self._lib, name)
        if not name.startswith("b200dp_") or name.endswith("_last_error") or name in PASS_THROUGH:
            return fn
        if name not in TABLE:
            def refuse(*args):
                raise GuardError(f"{name}: not in the launch table, so it may not run under the guard")
            return refuse

        def guarded(*args):
            check(name, args, self._blocks())
            self._calls[name] += 1
            return fn(*args)
        return guarded

    def __setattr__(self, name, value):
        setattr(self._lib, name, value)


GUARDED_MODULES = ("gemm", "bn", "ln", "conv", "attention", "dropout", "xent")


def install(monkeypatch):
    """Wrap the ``_lib`` of every binding module in ``GUARDED_MODULES``; returns the shared call counter."""
    import importlib
    calls = Counter()
    for m in GUARDED_MODULES:
        mod = importlib.import_module(f"distributed_torch_horovod_gcp_b200.ops.{m}")
        if mod._lib is not None:
            monkeypatch.setattr(mod, "_lib", GuardedLib(mod._lib, calls))
    return calls
