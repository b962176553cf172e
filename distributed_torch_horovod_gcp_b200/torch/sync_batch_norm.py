"""``hvd.SyncBatchNorm`` — batch norm with statistics reduced over all ranks.

Horovod surface parity (SURVEY.md §2.3, "not used by the reference").  Statistics
(sum, sum of squares, count) are packed into one small vector and all-reduced with the
framework's own ``allreduce`` (one-shot sm_90a kernel on CUDA: 2C+1 floats is a pure
latency message), forward and backward.

On H100 with NHWC bf16 activations the whole op runs on the fused BN kernels of
csrc/elementwise.cu with the NVLink allreduce BETWEEN their passes (``_SyncBNKernelFn``):
stats kernel -> one-shot allreduce -> finalize+apply kernel forward; masked-reduce kernel ->
one-shot allreduce -> dx kernel backward.  Other layouts / dtypes / CPU use the PyTorch composition
below (also the numerics oracle of the tests).
"""
from __future__ import annotations

import torch
from torch.nn.modules.batchnorm import _BatchNorm

from .. import _state
from . import mpi_ops


class _SyncBNFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, weight, bias, running_mean, running_var, eps, momentum):
        C = x.shape[1]
        dims = [0] + list(range(2, x.dim()))
        xf = x.float()
        n_local = x.numel() // C
        stats = torch.empty(2 * C + 1, dtype=torch.float32, device=x.device)
        stats[:C] = xf.sum(dims)
        stats[C:2 * C] = (xf * xf).sum(dims)
        stats[2 * C:].fill_(float(n_local))        # a fill kernel: item assignment would copy from the host
        stats = mpi_ops.allreduce(stats, op=mpi_ops.Sum, name=None)
        n = stats[2 * C]
        mean = stats[:C] / n
        var = (stats[C:2 * C] / n - mean * mean).clamp_min_(0.0)
        invstd = torch.rsqrt(var + eps)
        if running_mean is not None:
            with torch.no_grad():
                unbiased = var * (n / (n - 1).clamp_min(1.0))
                running_mean.mul_(1 - momentum).add_(mean.to(running_mean.dtype) * momentum)
                running_var.mul_(1 - momentum).add_(unbiased.to(running_var.dtype) * momentum)
        shape = [1, C] + [1] * (x.dim() - 2)
        xhat = (xf - mean.view(shape)) * invstd.view(shape)
        y = xhat
        if weight is not None:
            y = y * weight.float().view(shape)
        if bias is not None:
            y = y + bias.float().view(shape)
        ctx.save_for_backward(xhat, invstd, weight)
        ctx.n = n
        ctx.has_bias = bias is not None
        return y.to(x.dtype)

    @staticmethod
    def backward(ctx, dy):
        xhat, invstd, weight = ctx.saved_tensors
        C = xhat.shape[1]
        dims = [0] + list(range(2, xhat.dim()))
        shape = [1, C] + [1] * (xhat.dim() - 2)
        dyf = dy.float()
        sum_dy = dyf.sum(dims)
        sum_dy_xhat = (dyf * xhat).sum(dims)
        dweight = sum_dy_xhat.to(weight.dtype) if weight is not None else None
        dbias = sum_dy.to(weight.dtype if weight is not None else dy.dtype) \
            if ctx.has_bias else None
        packed = torch.cat([sum_dy, sum_dy_xhat])
        packed = mpi_ops.allreduce(packed, op=mpi_ops.Sum, name=None)
        g_sum_dy, g_sum_dy_xhat = packed[:C], packed[C:]
        w = weight.float().view(shape) if weight is not None else 1.0
        dx = (dyf - (g_sum_dy / ctx.n).view(shape)
              - xhat * (g_sum_dy_xhat / ctx.n).view(shape)) * invstd.view(shape) * w
        return dx.to(dy.dtype), dweight, dbias, None, None, None, None


class _SyncBNKernelFn(torch.autograd.Function):
    """NHWC bf16 SyncBN on the sm_90a BN kernels + one-shot allreduce of the per-channel sums."""

    @staticmethod
    def forward(ctx, x, weight, bias, running_mean, running_var, eps, momentum):
        from ..ops import bn as B
        lib = B._lib
        N, C, H, W = x.shape
        M = N * H * W
        dev = x.device
        st = torch.cuda.current_stream(dev).cuda_stream
        stats = torch.empty(2 * C + 1, dtype=torch.float32, device=dev)
        B._ck(lib.b200dp_bn_stats(x.data_ptr(), stats.data_ptr(), M, C, st))
        stats[2 * C:].fill_(float(M))           # a fill kernel: item assignment would copy from the host
        stats = mpi_ops.allreduce(stats, op=mpi_ops.Sum, name=None)
        count = stats[2 * C:]                   # global row count: ranks may hold different numbers of rows
        y = torch.empty_like(x, memory_format=torch.channels_last)
        ws = torch.empty(4 * C, dtype=torch.float32, device=dev)
        mean, invstd, a, b = ws[:C], ws[C:2 * C], ws[2 * C:3 * C], ws[3 * C:]
        B._ck(lib.b200dp_bn_fwd_sync(x.data_ptr(), None, y.data_ptr(), weight.data_ptr(), bias.data_ptr(),
                                     stats.data_ptr(), mean.data_ptr(), invstd.data_ptr(), a.data_ptr(),
                                     b.data_ptr(),
                                     running_mean.data_ptr() if running_mean is not None else None,
                                     running_var.data_ptr() if running_var is not None else None,
                                     M, count.data_ptr(), C, float(eps), float(momentum), 0,
                                     int(weight.dtype == torch.bfloat16), None, st))
        ctx.save_for_backward(x, mean, invstd, a, count)
        ctx.pdtype = weight.dtype
        return y

    @staticmethod
    def backward(ctx, dy):
        from ..ops import bn as B
        lib = B._lib
        x, mean, invstd, a, count = ctx.saved_tensors
        N, C, H, W = x.shape
        M = N * H * W
        if not dy.is_contiguous(memory_format=torch.channels_last):
            dy = dy.contiguous(memory_format=torch.channels_last)
        st = torch.cuda.current_stream(x.device).cuda_stream
        sums = torch.empty(2 * C, dtype=torch.float32, device=x.device)
        B._ck(lib.b200dp_bn_bwd_reduce(dy.data_ptr(), x.data_ptr(), None, mean.data_ptr(), sums.data_ptr(),
                                       M, C, 0, st))
        # parameter gradients are LOCAL sums (the DP optimizer averages them like any other gradient)
        dbeta = sums[:C].to(ctx.pdtype)
        dgamma = (sums[C:] * invstd).to(ctx.pdtype)
        g = mpi_ops.allreduce(sums, op=mpi_ops.Sum, name=None)
        dx = torch.empty_like(x, memory_format=torch.channels_last)
        B._ck(lib.b200dp_bn_bwd_apply(dy.data_ptr(), x.data_ptr(), None, dx.data_ptr(), None, a.data_ptr(),
                                      mean.data_ptr(), invstd.data_ptr(), g.data_ptr(), count.data_ptr(), M, C, 0,
                                      st))
        return dx, dgamma, dbeta, None, None, None, None


def _kernel_path_ok(x, weight, bias, running_mean=None, running_var=None) -> bool:
    if not (x.is_cuda and x.dim() == 4 and x.dtype == torch.bfloat16):
        return False
    try:
        from ..ops import kernels, bn as B
        # the kernels read (and write) every parameter in one dtype, chosen by `weight`
        if not B.params_ok(weight, bias, running_mean, running_var):
            return False
        if not kernels.has("bn_act") or not hasattr(B._lib, "b200dp_bn_fwd_sync"):
            return False
        return B.bn_supported(x, x.shape[1])
    except Exception:      # noqa: BLE001
        return False


class SyncBatchNorm(_BatchNorm):
    """Applies synchronous BatchNorm: statistics are computed over the global batch."""

    def _check_input_dim(self, input):
        if input.dim() < 2:
            raise ValueError("expected at least 2D input (got {}D input)".format(input.dim()))

    def forward(self, input):
        self._check_input_dim(input)
        if self.training and self.track_running_stats and self.num_batches_tracked is not None:
            self.num_batches_tracked.add_(1)
        momentum = self.momentum
        if momentum is None:
            momentum = 1.0 / float(self.num_batches_tracked) if self.track_running_stats else 0.0
        use_batch = self.training or not self.track_running_stats
        if not use_batch or not _state.is_initialized() or _state.size() == 1:
            return torch.nn.functional.batch_norm(
                input, self.running_mean, self.running_var, self.weight, self.bias,
                use_batch, momentum if momentum is not None else 0.0, self.eps)
        if _kernel_path_ok(input, self.weight, self.bias, self.running_mean, self.running_var):
            return _SyncBNKernelFn.apply(input, self.weight, self.bias, self.running_mean,
                                         self.running_var, self.eps, momentum)
        return _SyncBNFn.apply(input, self.weight, self.bias, self.running_mean,
                               self.running_var, self.eps, momentum)
