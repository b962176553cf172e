"""Tiny instances of every hand-written compute kernel, for compute-sanitizer:
    compute-sanitizer --tool racecheck|synccheck|memcheck python scripts/sanitize_kernels.py
Shapes are small (the tools slow kernels 10-100x) but cover: multi-tile persistent loops (several tiles per
CTA are not reachable at these sizes on 132 SMs, so max_ctas is forced down where the API allows), the
statistics / residual / masked-residual / split-K epilogues (per-CTA statistics slots, last-arriver split-K
reduction, fp32 and bf16 add / store outputs), 3x3 / strided / 1x1 conv paths incl. split-K wgrad, BN, LN, pooling, attention (non-causal and causal), the fused LM-head cross-entropy and the LSTM
recurrence, plus the fused engine's clip-by-global-norm kernels (reduce into R with norm slots, finalize, update) and its
LARS / LAMB kernels (reduce + direction + chunk partials, trust ratios + update)."""
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
# causal: the diagonal tile's mask, the shortened KV / query-tile loops and the reversed tile order
for S in (197, 300):
    q, k_, v = (rnd(2, 3, S, 64, scale=0.5).requires_grad_(True) for _ in range(3))
    kernels.attention_fused(q, k_, v, causal=True).float().sum().backward()
# fused LM-head cross-entropy: N and V not multiples of 128, an ignored row, 3 CTAs over several vocab ranges each,
# and 128-row backward chunks (the last one partial) with fp32 dW accumulation
from distributed_torch_horovod_gcp_b200.ops import xent as XE
XE._CHUNK_BYTES = 2 * 128 * 1000
xx, ww = rnd(300, 64).requires_grad_(True), rnd(1000, 64, scale=0.2).requires_grad_(True)
tt = torch.randint(0, 1000, (300,), device=dev)
tt[5] = -100
XE.linear_cross_entropy(xx, ww, tt, max_ctas=3).backward()
XE.linear_cross_entropy(xx, ww, tt, reduction="none", max_ctas=3).sum().backward()
print("xent ok", float(xx.grad.float().abs().sum()))
from distributed_torch_horovod_gcp_b200.models import LSTM
m = LSTM(23, 20, 1, 256, device=torch.device(dev)).to(dev)
xs = torch.randn(8, 20, 23, device=dev)
m(xs).sum().backward()
# stacked bidirectional: reverse direction, strided halves of seq, F > 32 input products with a tail
m2 = LSTM(40, 5, 1, 256, n_layers=2, bidirectional=True, device=torch.device(dev)).to(dev)
m2(torch.randn(7, 5, 40, device=dev)).sum().backward()
# inter-layer dropout: the mask kernel and the dropped-input products of the layers above the first
m3 = LSTM(40, 5, 1, 256, n_layers=3, bidirectional=True, dropout=0.3, device=torch.device(dev)).to(dev)
m3(torch.randn(7, 5, 40, device=dev)).sum().backward()
torch.cuda.synchronize()

# fused engine in clip mode on one GPU: several buckets, bf16 parameters with fp32 masters, two steps
os.environ["B200DP_FUSED_SINGLE"] = "1"
import distributed_torch_horovod_gcp_b200.torch as hvd
hvd.init()
mlp = nn.Sequential(nn.Linear(32, 100), nn.ReLU(), nn.Linear(100, 7)).to(dev).to(bf)
opt = hvd.DistributedOptimizer(torch.optim.Adam(mlp.parameters(), lr=1e-3), named_parameters=mlp.named_parameters(),
                               bucket_bytes=4096, max_grad_norm=0.01)
assert opt.fused_engine is not None and opt.fused_engine.clip
for _ in range(2):
    mlp(rnd(8, 32)).float().square().mean().backward()
    opt.step()
    opt.zero_grad()
torch.cuda.synchronize()
print("clip ok", float(opt.grad_norm))
# LARS / LAMB: reduce + direction + chunk partials, then ratios + update; bf16 buckets of several tensors, and
# an fp32 tensor of several chunks shared by several CTAs
for kind, dt, width in (("lamb", bf, 100), ("lars", torch.float32, 400)):
    net = nn.Sequential(nn.Linear(96, width), nn.ReLU(), nn.Linear(width, 7)).to(dev).to(dt)
    groups = [{"params": [p for p in net.parameters() if p.dim() > 1]},
              {"params": [p for p in net.parameters() if p.dim() == 1], "weight_decay": 0.0, "adaptive": False}]
    base = hvd.LAMB(groups, lr=1e-3) if kind == "lamb" else hvd.LARS(groups, lr=0.1, weight_decay=1e-4)
    opt = hvd.DistributedOptimizer(base, named_parameters=net.named_parameters(), bucket_bytes=4096)
    assert opt.fused_engine is not None and opt.fused_engine.layerwise
    for _ in range(2):
        net(torch.randn(8, 96, device=dev, dtype=dt)).float().square().mean().backward()
        opt.step()
        opt.zero_grad()
    torch.cuda.synchronize()
    print(kind, "ok", float(opt.fused_engine.lw_ratio.sum()))
hvd.shutdown()
print("all ok")
