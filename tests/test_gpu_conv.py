"""Implicit-GEMM convolution (csrc/conv_sm90.cu) vs an fp32 PyTorch reference of the same op:
forward, data gradient and weight gradient for every ResNet shape class (3x3 s1, 3x3 s2, 1x1 s2),
including pixel spaces that do not tile evenly (odd batch, 7x7 / 14x14 maps)."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


def _kern():
    from distributed_torch_horovod_gcp_b200.ops import kernels
    assert kernels.has("conv_implicit_gemm"), "conv kernel missing from libb200dp_kernels.so"
    return kernels


def _rel(a, b):
    return ((a.float() - b.float()).norm() / b.float().norm().clamp_min(1e-6)).item()


CASES = [
    # N, Cin, H, W, Cout, R, stride
    (8, 64, 56, 56, 64, 3, 1),
    (4, 128, 28, 28, 128, 3, 1),
    (4, 256, 28, 28, 256, 3, 2),
    (2, 512, 7, 7, 512, 3, 1),
    (3, 256, 14, 14, 256, 3, 1),       # odd batch, 14x14 -> boxes clipped in N
    (5, 128, 56, 56, 128, 3, 2),
    (4, 256, 56, 56, 512, 1, 2),       # downsample 1x1 stride 2
    (2, 1024, 14, 14, 2048, 1, 2),
    (2, 64, 20, 12, 96, 3, 1),         # spatial extent that is not a power-of-two multiple
    (2, 512, 14, 14, 512, 3, 2),
]


@pytest.mark.parametrize("N,C,H,W,K,R,stride", CASES)
def test_conv_matches_fp32_reference(N, C, H, W, K, R, stride):
    k = _kern()
    torch.manual_seed(0)
    pad = (R - 1) // 2
    x = torch.randn(N, C, H, W, device="cuda").to(torch.bfloat16).contiguous(
        memory_format=torch.channels_last).requires_grad_(True)
    w = (torch.randn(K, C, R, R, device="cuda") * 0.05).to(torch.bfloat16).contiguous(
        memory_format=torch.channels_last).requires_grad_(True)
    xr, wr = x.detach().float().requires_grad_(True), w.detach().float().requires_grad_(True)
    y = k.conv2d_implicit(x, w, stride, pad)
    yr = F.conv2d(xr, wr, None, stride, pad)
    assert y.shape == yr.shape
    assert y.is_contiguous(memory_format=torch.channels_last)
    assert _rel(y, yr) < 8e-3
    g = torch.randn_like(y)
    y.backward(g)
    yr.backward(g.float())
    assert _rel(x.grad, xr.grad) < 1.5e-2
    assert _rel(w.grad, wr.grad) < 1.5e-2
    # second backward through a fresh graph: no state from the first weight gradient may leak into it
    x.grad = None
    w.grad = None
    y2 = k.conv2d_implicit(x, w, stride, pad)
    y2.backward(g)
    assert _rel(w.grad, wr.grad) < 1.5e-2


def test_conv_default_layout_weight():
    """A weight in the default (NCHW-contiguous) layout is re-laid-out on the fly."""
    k = _kern()
    torch.manual_seed(1)
    x = torch.randn(2, 64, 16, 16, device="cuda").to(torch.bfloat16).contiguous(
        memory_format=torch.channels_last)
    w = (torch.randn(64, 64, 3, 3, device="cuda") * 0.05).to(torch.bfloat16).requires_grad_(True)
    y = k.conv2d_implicit(x, w, 1, 1)
    yr = F.conv2d(x.float(), w.float(), None, 1, 1)
    assert _rel(y, yr) < 8e-3
    y.sum().backward()
    assert w.grad is not None and w.grad.shape == w.shape


def test_resnet_block_uses_no_cudnn_conv():
    """ResNet bottleneck + basic block forward/backward: every conv goes through our kernels."""
    from distributed_torch_horovod_gcp_b200.models.resnet import Bottleneck, BasicBlock
    from distributed_torch_horovod_gcp_b200.ops import counters
    import torch.nn as nn
    torch.manual_seed(2)
    ds = nn.Sequential(nn.Conv2d(64, 512, 1, 2, bias=False), nn.BatchNorm2d(512))
    blk = Bottleneck(64, 128, stride=2, downsample=ds).cuda().to(torch.bfloat16).to(
        memory_format=torch.channels_last)
    x = torch.randn(4, 64, 28, 28, device="cuda").to(torch.bfloat16).contiguous(
        memory_format=torch.channels_last).requires_grad_(True)
    c0 = dict(counters.snapshot()) if hasattr(counters, "snapshot") else None
    y = blk(x)
    y.float().mean().backward()
    assert x.grad is not None and torch.isfinite(x.grad.float()).all()
    if c0 is not None:
        c1 = counters.snapshot()
        assert c1.get("conv_fprop", 0) - c0.get("conv_fprop", 0) == 2      # 3x3 s2 + 1x1 s2 downsample
        assert c1.get("conv_dgrad", 0) - c0.get("conv_dgrad", 0) >= 2
    bb = BasicBlock(64, 64).cuda().to(torch.bfloat16).to(memory_format=torch.channels_last)
    yb = bb(x.detach())
    yb.float().mean().backward()


def test_grad_sink_matches_autograd_path():
    """Weight gradients written straight into the gradient buckets (ops/grad_sink.py) == the same
    backward through autograd's AccumulateGrad.  The forward is deterministic, so the two gradient
    sets must agree to the rounding of the paths that convert and accumulate them."""
    import os
    os.environ["B200DP_FUSED_SINGLE"] = "1"
    import torch.nn as nn
    import distributed_torch_horovod_gcp_b200.torch as hvd
    from distributed_torch_horovod_gcp_b200.ops import grad_sink, functional as F2, kernels

    class Net(nn.Module):
        def __init__(self):
            super().__init__()
            self.c1 = nn.Conv2d(16, 64, 3, 1, 1, bias=False)
            self.c2 = nn.Conv2d(64, 128, 3, 2, 1, bias=False)
            self.c3 = nn.Conv2d(128, 256, 1, 2, 0, bias=False)
            self.c4 = nn.Conv2d(256, 256, 1, 1, 0, bias=False)
            self.fc = nn.Linear(256, 16)

        def forward(self, x):
            from distributed_torch_horovod_gcp_b200.ops.bn import conv2d
            for c in (self.c1, self.c2, self.c3, self.c4):
                x = torch.relu(conv2d(x, c)[0])
            return F2.linear(x.mean(dim=(2, 3)), self.fc.weight, self.fc.bias)

    hvd.init()
    kernels.has("conv_implicit_gemm")
    grads = []
    for enabled in (True, False):
        grad_sink._ENABLED = enabled
        torch.manual_seed(0)
        model = Net().cuda().to(torch.bfloat16).to(memory_format=torch.channels_last)
        opt = hvd.DistributedOptimizer(torch.optim.SGD(model.parameters(), lr=0.05, momentum=0.9),
                                       named_parameters=model.named_parameters(),
                                       backward_passes_per_step=3)
        assert opt.fused_engine is not None
        x = torch.randn(8, 16, 32, 32, device="cuda").to(torch.bfloat16).contiguous(
            memory_format=torch.channels_last)
        y = torch.randint(0, 16, (8,), device="cuda")
        F.cross_entropy(model(x).float(), y).backward()      # pass 1 of 3: gradients stay in the buckets
        torch.cuda.synchronize()
        g1 = {n: p.grad.detach().float().clone() for n, p in model.named_parameters()}
        F.cross_entropy(model(x).float(), y).backward()      # pass 2 accumulates on top (accumulate path)
        torch.cuda.synchronize()
        g2 = {n: p.grad.detach().float().clone() for n, p in model.named_parameters()}
        F.cross_entropy(model(x).float(), y).backward()      # pass 3 launches the buckets
        opt.step()
        opt.zero_grad()
        torch.cuda.synchronize()
        grads.append((g1, g2))
        opt.remove_hooks()
    grad_sink._ENABLED = True
    hvd.shutdown()
    (a1, a2), (b1, b2) = grads
    for n in a1:
        assert a1[n].abs().sum() > 0, n
        assert _rel(a1[n], b1[n]) < 1e-2, (n, _rel(a1[n], b1[n]))
        assert _rel(a2[n], b2[n]) < 1e-2, (n, _rel(a2[n], b2[n]))
        assert _rel(a2[n], 2 * a1[n]) < 2e-2, n


@pytest.mark.parametrize("kind", ["identity", "projection_s1", "projection_s2"])
def test_bottleneck_skip_gradient_goes_through_dgrad_epilogue(kind):
    """The block input feeds conv1 and the skip branch; its second gradient is added by conv1's dgrad GEMM
    epilogue (ops.grad_sink.GradBox) — identity block: bn3's unmasked dy + ReLU sign bits; projection block:
    the downsample conv's dgrad, with the sign bits handed to the downsample BN.  Oracle: the same kernels
    with the boxes disabled (autograd's stand-alone add, masked copy written by the BN backward), plus a
    loose check against the fp32 reference composition."""
    import copy
    import torch.nn as nn
    from distributed_torch_horovod_gcp_b200.models.resnet import Bottleneck
    from distributed_torch_horovod_gcp_b200.ops import functional as F2
    _kern()
    torch.manual_seed(4)
    if kind == "identity":
        blk, cin, hw = Bottleneck(256, 64), 256, 14
    else:
        stride = 1 if kind == "projection_s1" else 2
        ds = nn.Sequential(nn.Conv2d(128, 256, 1, stride, bias=False), nn.BatchNorm2d(256))
        blk, cin, hw = Bottleneck(128, 64, stride, ds), 128, 28
    blk = blk.cuda().to(torch.bfloat16).to(memory_format=torch.channels_last)
    ref = copy.deepcopy(blk).float()
    x0 = torch.randn(8, cin, hw, hw, device="cuda").to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
    with torch.no_grad():
        oshape = blk(x0).shape
    g = torch.randn(oshape, device="cuda").to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
    grads, wgrads = [], []
    real_box = F2.new_grad_box
    for use_box in (True, False, True):
        F2.new_grad_box = real_box if use_box else (lambda t: None)
        try:
            # x is an intermediate (as in the network), so that a withheld gradient would go missing
            leaf = x0.clone().requires_grad_(True)
            x = leaf * 1.0
            blk.zero_grad()
            blk(x).backward(g)
            grads.append(leaf.grad.float().clone())
            wgrads.append(blk.conv1.weight.grad.float().clone())
        finally:
            F2.new_grad_box = real_box
    assert _rel(grads[0], grads[1]) < 1e-2          # fused add == stand-alone add
    assert _rel(grads[2], grads[1]) < 1e-2          # the box is per-forward state: second use is clean
    assert _rel(wgrads[0], wgrads[1]) < 1e-2
    xr = x0.detach().float().requires_grad_(True)
    F2._FORCE_REFERENCE = True
    try:
        ref(xr).backward(g.float())
    finally:
        F2._FORCE_REFERENCE = False
    assert _rel(grads[0], xr.grad) < 1e-1           # bf16 activations / BN statistics vs fp32 end to end


def test_gemm_masked_residual():
    """dgrad GEMM with a bit-masked residual (C = A B + mask(R)): the skip gradient of an identity block
    is bn3's incoming gradient with the block's ReLU sign bits (1 byte / 8 channels) applied in the epilogue."""
    from distributed_torch_horovod_gcp_b200.ops import gemm as G
    _kern()
    torch.manual_seed(9)
    M, N, K = 1000, 256, 64
    a = torch.randn(M, K, device="cuda").to(torch.bfloat16)
    b = (torch.randn(N, K, device="cuda") * 0.1).to(torch.bfloat16)
    r = torch.randn(M, N, device="cuda").to(torch.bfloat16)
    keep = torch.rand(M, N, device="cuda") > 0.5
    bits = (keep.view(M, N // 8, 8).to(torch.uint8) << torch.arange(8, device="cuda", dtype=torch.uint8)).sum(
        dim=2).to(torch.uint8).contiguous()
    out = torch.empty(M, N, device="cuda", dtype=torch.bfloat16)
    G.gemm(a, b, out, M, N, K, residual=r, res_mask=bits)
    ref = a.float() @ b.float().t() + r.float() * keep.float()
    assert _rel(out.float(), ref) < 1e-2
    G.gemm(a, b, out, M, N, K, residual=r)
    assert _rel(out.float(), a.float() @ b.float().t() + r.float()) < 1e-2


@pytest.mark.parametrize("cin,cout,k,stride,hw", [(64, 256, 1, 1, 28), (64, 64, 3, 1, 28), (128, 256, 3, 1, 14),
                                                 (128, 128, 3, 2, 28), (256, 512, 1, 2, 28), (3, 64, 7, 2, 64),
                                                 (256, 2048, 1, 1, 7)])
def test_bn_statistics_from_conv_epilogue(cin, cout, k, stride, hw):
    """conv+BN(+ReLU) with the batch statistics accumulated by the conv / GEMM epilogue == the same unit
    with the stand-alone statistics pass, for every convolution path (GEMM, implicit GEMM,
    strided, stem), twice in a row (the persistent accumulator is re-zeroed by the finalize kernel)."""
    import torch.nn as nn
    from distributed_torch_horovod_gcp_b200.ops import bn as B
    _kern()
    torch.manual_seed(6)
    conv = nn.Conv2d(cin, cout, k, stride, (k - 1) // 2, bias=False).cuda().to(torch.bfloat16).to(
        memory_format=torch.channels_last)
    bns = [nn.BatchNorm2d(cout).cuda().to(torch.bfloat16) for _ in range(2)]
    x = torch.randn(8, cin, hw, hw, device="cuda").to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
    outs = []
    for fuse, bn in zip((True, False), bns):
        B._FUSE_STATS = fuse
        try:
            for _ in range(2):
                y = B.conv_bn_act(x, conv, bn, relu=True)
        finally:
            B._FUSE_STATS = True
        outs.append((y.float(), bn.running_mean.float().clone(), bn.running_var.float().clone()))
    (ya, ma, va), (yb, mb, vb) = outs
    assert hasattr(bns[0], "_b200dp_stats") and float(bns[0]._b200dp_stats.abs().sum()) == 0.0
    assert _rel(ya, yb) < 5e-3
    assert _rel(ma, mb) < 1e-3 and _rel(va, vb) < 1e-3
