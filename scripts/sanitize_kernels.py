"""Tiny instances of every hand-written compute kernel, for compute-sanitizer:
    compute-sanitizer --tool racecheck|synccheck|memcheck python scripts/sanitize_kernels.py
Shapes are small (the tools slow kernels 10-100x) but cover: multi-tile persistent loops (several tiles per
CTA are not reachable at these sizes on 132 SMs, so max_ctas is forced down where the API allows), the
statistics / residual / masked-residual / split-K epilogues (per-CTA statistics slots, last-arriver split-K
reduction, fp32 and bf16 add / store outputs), 3x3 / strided / 1x1 conv paths incl. split-K wgrad, BN, LN, pooling, attention and the LSTM
recurrence."""
import os, sys, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from distributed_torch_horovod_gcp_b200.ops import kernels, gemm as G, conv as C, bn as B
import torch.nn as nn
assert kernels.has("conv_implicit_gemm")
dev = "cuda"
torch.manual_seed(0)
bf = torch.bfloat16

def rnd(*s, scale=1.0):
    return (torch.randn(*s, device=dev) * scale).to(bf)

# GEMM: plain+stats, residual, masked residual, split-K fp32 accumulate; few CTAs -> several tiles each
M, N, K = 1536, 256, 128
a, b, r = rnd(M, K), rnd(N, K, scale=0.1), rnd(M, N)
out = torch.empty(M, N, device=dev, dtype=bf)
stats = torch.zeros(2 * N, device=dev)
G.gemm(a, b, out, M, N, K, stats=stats, max_ctas=4)
G.gemm(a, b, out, M, N, K, residual=r, max_ctas=4)
bits = torch.randint(0, 256, (M, N // 8), device=dev, dtype=torch.uint8)
G.gemm(a, b, out, M, N, K, residual=r, res_mask=bits, max_ctas=4)
acc = torch.zeros(N, K, device=dev)
G.gemm(out, a, acc, N, K, M, a_mn=True, b_mn=True, out_mode=1, splits=4)
# the same into a bf16 C: split-K store, then a single-split add (no atomics, one writer per element)
acc16 = torch.empty(N, K, device=dev, dtype=bf)
G.gemm(out, a, acc16, N, K, M, a_mn=True, b_mn=True, out_mode=2, splits=4)
G.gemm(out, a, acc16, N, K, M, a_mn=True, b_mn=True, out_mode=1, max_ctas=1)
print("gemm ok", float(out.float().abs().mean()))

# convolutions: 64 / 256 ch, strided, 1x1, with BN statistics; dgrad + wgrad (split-K) through autograd
for cin, cout, k, s, hw in ((64, 64, 3, 1, 16), (256, 256, 3, 1, 8), (128, 128, 3, 2, 16), (256, 512, 1, 2, 8)):
    conv = nn.Conv2d(cin, cout, k, s, (k - 1) // 2, bias=False).to(dev).to(bf).to(memory_format=torch.channels_last)
    bn = nn.BatchNorm2d(cout).to(dev).to(bf)
    x = rnd(4, cin, hw, hw).contiguous(memory_format=torch.channels_last).requires_grad_(True)
    y = B.conv_bn_act(x, conv, bn, relu=True)
    y.float().square().mean().backward()
print("conv+bn ok")

# pooling, LN, attention, LSTM recurrence (through the public functional layer)
from distributed_torch_horovod_gcp_b200.ops import functional as F2
x = rnd(2, 64, 16, 16).contiguous(memory_format=torch.channels_last).requires_grad_(True)
F2.global_avg_pool(F2.max_pool_3x3_s2(x)).float().sum().backward()
ln = nn.LayerNorm(256).to(dev).to(bf)
t = rnd(64, 256).requires_grad_(True)
F2.layer_norm(t, ln.weight, ln.bias).float().sum().backward()
q, k_, v = (rnd(2, 4, 197, 64, scale=0.5).requires_grad_(True) for _ in range(3))
kernels.attention_fused(q, k_, v).float().sum().backward()
from distributed_torch_horovod_gcp_b200.models import LSTM
m = LSTM(23, 20, 1, 256, device=torch.device(dev)).to(dev)
xs = torch.randn(8, 20, 23, device=dev)
m(xs).sum().backward()
torch.cuda.synchronize()
print("all ok")
