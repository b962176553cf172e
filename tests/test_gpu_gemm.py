"""wgmma GEMM (csrc/gemm_sm90.cu) vs a plain PyTorch fp32 reference of the same op."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _k():
    from distributed_torch_horovod_gcp_b200.ops import kernels, gemm
    assert kernels.has("gemm"), "libb200dp_kernels.so not loaded / gemm symbol missing"
    return gemm


def _rel(a, b):
    return ((a.float() - b.float()).norm() / b.float().norm().clamp_min(1e-6)).item()


@pytest.mark.parametrize("M,N,K", [(128, 64, 64), (256, 256, 512), (1000, 384, 200), (4096, 1024, 1024),
                                   (50176, 64, 256), (197 * 8, 2304, 768), (33, 8, 72)])
@pytest.mark.parametrize("bn", [0, 64, 128, 256])
def test_gemm_kmajor(M, N, K, bn):
    g = _k()
    torch.manual_seed(0)
    a = torch.randn(M, K, device="cuda", dtype=torch.bfloat16)
    b = torch.randn(N, K, device="cuda", dtype=torch.bfloat16)
    out = torch.empty(M, N, device="cuda", dtype=torch.bfloat16)
    g.gemm(a, b, out, M, N, K, block_n=bn)
    ref = a.float() @ b.float().t()
    assert _rel(out, ref) < 6e-3


@pytest.mark.parametrize("a_mn,b_mn", [(False, True), (True, False), (True, True)])
@pytest.mark.parametrize("M,N,K", [(256, 128, 512), (1024, 200, 328), (64, 64, 4096)])
def test_gemm_mn_major(a_mn, b_mn, M, N, K):
    g = _k()
    torch.manual_seed(1)
    A = torch.randn(M, K, device="cuda", dtype=torch.bfloat16)
    B = torch.randn(N, K, device="cuda", dtype=torch.bfloat16)
    a = A.t().contiguous() if a_mn else A            # [K, M] when MN-major
    b = B.t().contiguous() if b_mn else B
    if (a_mn and M % 8) or (b_mn and N % 8):
        pytest.skip("MN-major needs the row count to be a multiple of 8")
    out = torch.empty(M, N, device="cuda", dtype=torch.bfloat16)
    g.gemm(a, b, out, M, N, K, a_mn=a_mn, b_mn=b_mn)
    assert _rel(out, A.float() @ B.float().t()) < 6e-3


def test_gemm_epilogues_and_splitk():
    g = _k()
    torch.manual_seed(2)
    M, N, K = 512, 384, 640
    a = torch.randn(M, K, device="cuda", dtype=torch.bfloat16) * 0.1
    b = torch.randn(N, K, device="cuda", dtype=torch.bfloat16)
    bias = torch.randn(N, device="cuda", dtype=torch.bfloat16)
    res = torch.randn(M, N, device="cuda", dtype=torch.bfloat16)
    ref0 = a.float() @ b.float().t() + bias.float()
    for act, fn in ((1, torch.relu), (2, torch.nn.functional.gelu)):
        out = torch.empty(M, N, device="cuda", dtype=torch.bfloat16)
        z = torch.empty_like(out)
        g.gemm(a, b, out, M, N, K, bias=bias, residual=res, preact=z, act=act)
        assert _rel(out, fn(ref0) + res.float()) < 8e-3
        assert _rel(z, ref0) < 8e-3
    # fp32 bias, fp32 store
    o32 = torch.empty(M, N, device="cuda", dtype=torch.float32)
    g.gemm(a, b, o32, M, N, K, bias=bias.float(), out_mode=2)
    assert _rel(o32, ref0) < 2e-3
    # split-K with fp32 atomics accumulates on top of existing contents
    acc = torch.ones(M, N, device="cuda", dtype=torch.float32)
    g.gemm(a, b, acc, M, N, K, out_mode=1, splits=5)
    assert _rel(acc, a.float() @ b.float().t() + 1.0) < 2e-3
    # backward-activation epilogues
    aux = torch.randn(M, N, device="cuda", dtype=torch.bfloat16)
    out = torch.empty(M, N, device="cuda", dtype=torch.bfloat16)
    g.gemm(a, b, out, M, N, K, residual=aux, act=4)
    assert _rel(out, (a.float() @ b.float().t()) * (aux.float() > 0)) < 8e-3


def test_linear_autograd_matches_torch():
    from distributed_torch_horovod_gcp_b200.ops import functional as F2
    torch.manual_seed(3)
    x = torch.randn(4, 197, 768, device="cuda", dtype=torch.bfloat16, requires_grad=True)
    w = (torch.randn(3072, 768, device="cuda", dtype=torch.bfloat16) * 0.03).requires_grad_(True)
    b = torch.randn(3072, device="cuda", dtype=torch.bfloat16, requires_grad=True)
    xr, wr, br = [t.detach().float().requires_grad_(True) for t in (x, w, b)]
    y = F2.linear(x, w, b, act="gelu")
    yr = torch.nn.functional.gelu(torch.nn.functional.linear(xr, wr, br))
    assert _rel(y, yr) < 1e-2
    gy = torch.randn_like(y)
    y.backward(gy)
    yr.backward(gy.float())
    assert _rel(x.grad, xr.grad) < 2e-2
    assert _rel(w.grad, wr.grad) < 2e-2
    assert _rel(b.grad, br.grad) < 2e-2
    from distributed_torch_horovod_gcp_b200.ops import counters
    assert counters.snapshot().get("gemm_sm90", 0) >= 3


@pytest.mark.parametrize("C,relu,res", [(64, True, False), (256, True, True), (2048, False, False),
                                        (128, False, True)])
def test_fused_bn_matches_torch(C, relu, res):
    from distributed_torch_horovod_gcp_b200.ops import kernels
    assert kernels.has("bn_act")
    torch.manual_seed(4)
    N, H, W = 8, 14, 14
    x = torch.randn(N, C, H, W, device="cuda").to(torch.bfloat16).contiguous(
        memory_format=torch.channels_last).requires_grad_(True)
    r = torch.randn(N, C, H, W, device="cuda").to(torch.bfloat16).contiguous(
        memory_format=torch.channels_last).requires_grad_(True) if res else None
    bn = torch.nn.BatchNorm2d(C).cuda().to(torch.bfloat16)
    with torch.no_grad():
        bn.weight.copy_(torch.rand(C) + 0.5)
        bn.bias.copy_(torch.randn(C) * 0.1)
    ref = torch.nn.BatchNorm2d(C).cuda()
    with torch.no_grad():
        ref.weight.copy_(bn.weight.float())
        ref.bias.copy_(bn.bias.float())
    y = kernels.bn_act(x, bn, relu, r)
    xr = x.detach().float().requires_grad_(True)
    rr = r.detach().float().requires_grad_(True) if res else None
    yr = ref(xr)
    if res:
        yr = yr + rr
    if relu:
        yr = torch.relu(yr)
    assert _rel(y, yr) < 1e-2
    gy = torch.randn_like(y)
    y.backward(gy)
    yr.backward(gy.float())
    assert _rel(x.grad, xr.grad) < 2e-2
    assert _rel(bn.weight.grad, ref.weight.grad) < 2e-2
    assert _rel(bn.bias.grad, ref.bias.grad) < 2e-2
    if res:
        assert _rel(r.grad, rr.grad) < 1e-2
    assert _rel(bn.running_var, ref.running_var) < 2e-2
    assert _rel(bn.running_mean + 1.0, ref.running_mean + 1.0) < 1e-2


def test_resnet50_kernels_vs_reference_ops():
    """Whole-model check: the kernel path (wgmma 1x1 convs + fused BN) must be as close to an
    fp32 run of the same model as the library bf16 path is (bf16 noise through 53 BN layers is
    large, so the two bf16 paths are each compared with the fp32 oracle, not with each other)."""
    import copy
    from distributed_torch_horovod_gcp_b200.models import resnet50
    from distributed_torch_horovod_gcp_b200.ops import functional as F2
    torch.manual_seed(5)
    m32 = resnet50(num_classes=64).cuda().to(memory_format=torch.channels_last)
    m = copy.deepcopy(m32).to(torch.bfloat16)
    x32 = torch.randn(32, 3, 64, 64, device="cuda").contiguous(memory_format=torch.channels_last)
    x = x32.to(torch.bfloat16)
    F2._FORCE_REFERENCE = True
    try:
        y32 = m32(x32)
        y32.sum().backward()
        yr = m(x)
        yr.float().sum().backward()
        gr = m.fc.weight.grad.clone()
        cr = m.layer1[0].conv1.weight.grad.clone()
    finally:
        F2._FORCE_REFERENCE = False
    m.zero_grad()
    y = m(x)
    y.float().sum().backward()
    e_ref, e_ker = _rel(yr, y32), _rel(y, y32)
    print("fwd rel err vs fp32: library", e_ref, "kernels", e_ker)
    assert e_ker < max(2.0 * e_ref, 0.05)
    g_ref, g_ker = _rel(gr, m32.fc.weight.grad), _rel(m.fc.weight.grad, m32.fc.weight.grad)
    c_ref, c_ker = _rel(cr, m32.layer1[0].conv1.weight.grad), \
        _rel(m.layer1[0].conv1.weight.grad, m32.layer1[0].conv1.weight.grad)
    print("grad rel err vs fp32: fc", g_ref, g_ker, "layer1.0.conv1", c_ref, c_ker)
    assert g_ker < max(2.0 * g_ref, 0.05)
    assert c_ker < max(2.5 * c_ref, 0.1)


def test_maxpool_matches_torch():
    from distributed_torch_horovod_gcp_b200.ops import kernels
    assert kernels.has("max_pool_3x3_s2")
    torch.manual_seed(6)
    for (N, C, H, W) in [(4, 64, 112, 112), (2, 16, 9, 7)]:
        x = torch.randn(N, C, H, W, device="cuda").to(torch.bfloat16).contiguous(
            memory_format=torch.channels_last).requires_grad_(True)
        xr = x.detach().float().requires_grad_(True)
        y = kernels.max_pool_3x3_s2(x)
        yr = torch.nn.functional.max_pool2d(xr, 3, 2, 1)
        assert torch.equal(y.float(), yr)
        g = torch.randn_like(y)
        y.backward(g)
        yr.backward(g.float())
        # ties are measure-zero for random inputs; bf16 accumulation of <= 4 terms
        assert _rel(x.grad, xr.grad) < 1e-2


def test_stem_conv_matches_cudnn():
    from distributed_torch_horovod_gcp_b200.ops import kernels, bn as B
    assert kernels.has("stem_conv")
    torch.manual_seed(8)
    conv = torch.nn.Conv2d(3, 64, 7, 2, 3, bias=False).cuda().to(torch.bfloat16).to(
        memory_format=torch.channels_last)
    x = torch.randn(4, 3, 64, 96, device="cuda").to(torch.bfloat16).contiguous(
        memory_format=torch.channels_last)
    assert B._is_stem_conv(x, conv)
    y = B.conv2d(x, conv)[0]
    ref = torch.nn.functional.conv2d(x.float(), conv.weight.float(), None, 2, 3)
    assert y.shape == ref.shape and _rel(y, ref) < 6e-3
    gy = torch.randn_like(y)
    y.backward(gy)
    wr = conv.weight.detach().float().requires_grad_(True)
    torch.nn.functional.conv2d(x.float(), wr, None, 2, 3).backward(gy.float())
    assert _rel(conv.weight.grad, wr.grad) < 1e-2


def test_mlp_block_matches_torch():
    from distributed_torch_horovod_gcp_b200.ops import functional as F2
    torch.manual_seed(9)
    x = (torch.randn(2, 197, 768, device="cuda") * 0.5).to(torch.bfloat16).requires_grad_(True)
    w1 = (torch.randn(3072, 768, device="cuda") * 0.03).to(torch.bfloat16).requires_grad_(True)
    b1 = (torch.randn(3072, device="cuda") * 0.1).to(torch.bfloat16).requires_grad_(True)
    w2 = (torch.randn(768, 3072, device="cuda") * 0.02).to(torch.bfloat16).requires_grad_(True)
    b2 = (torch.randn(768, device="cuda") * 0.1).to(torch.bfloat16).requires_grad_(True)
    ts = (x, w1, b1, w2, b2)
    rs = [t.detach().float().requires_grad_(True) for t in ts]
    y = F2.mlp(x, w1, b1, w2, b2, residual=x)
    yr = torch.nn.functional.linear(torch.nn.functional.gelu(torch.nn.functional.linear(rs[0], rs[1], rs[2])),
                                    rs[3], rs[4]) + rs[0]
    assert _rel(y, yr) < 1e-2
    g = torch.randn_like(y)
    y.backward(g)
    yr.backward(g.float())
    for t, r, name in zip(ts, rs, "x w1 b1 w2 b2".split()):
        assert _rel(t.grad, r.grad) < 3e-2, name


@pytest.mark.parametrize("R,C", [(25216, 768), (128, 768), (1000, 1024), (33, 256)])
def test_layer_norm_matches_torch(R, C):
    from distributed_torch_horovod_gcp_b200.ops import kernels
    assert kernels.has("layer_norm")
    torch.manual_seed(10)
    x = (torch.randn(R, C, device="cuda") * 2 + 0.5).to(torch.bfloat16).requires_grad_(True)
    w = (torch.rand(C, device="cuda") + 0.5).to(torch.bfloat16).requires_grad_(True)
    b = (torch.randn(C, device="cuda") * 0.1).to(torch.bfloat16).requires_grad_(True)
    xr, wr, br = [t.detach().float().requires_grad_(True) for t in (x, w, b)]
    y = kernels.layer_norm(x, w, b, 1e-6)
    yr = torch.nn.functional.layer_norm(xr, (C,), wr, br, 1e-6)
    assert _rel(y, yr) < 1e-2
    g = torch.randn_like(y)
    y.backward(g)
    yr.backward(g.float())
    assert _rel(x.grad, xr.grad) < 2e-2
    assert _rel(w.grad, wr.grad) < 2e-2
    assert _rel(b.grad, br.grad) < 2e-2


@pytest.mark.parametrize("a_mn,b_mn", [(False, False), (False, True), (True, True), (True, False)])
@pytest.mark.parametrize("M,N,K", [(512, 256, 256), (25216, 768, 3072), (1000, 2304, 768), (4096, 264, 512)])
def test_gemm_large_operand_layouts(a_mn, b_mn, M, N, K):
    """Wide / deep GEMMs (ViT-B shapes among them) in every operand layout, direct and split-K."""
    g = _k()
    torch.manual_seed(11)
    A = torch.randn(M, K, device="cuda", dtype=torch.bfloat16) * 0.5
    B = torch.randn(N, K, device="cuda", dtype=torch.bfloat16) * 0.5
    a = A.t().contiguous() if a_mn else A
    b = B.t().contiguous() if b_mn else B
    if (a_mn and M % 8) or (b_mn and N % 8):
        pytest.skip("MN-major needs the row count to be a multiple of 8")
    out = torch.empty(M, N, device="cuda", dtype=torch.bfloat16)
    g.gemm(a, b, out, M, N, K, a_mn=a_mn, b_mn=b_mn)
    assert _rel(out, A.float() @ B.float().t()) < 6e-3
    # split-K + fp32 accumulation
    acc = torch.zeros(M, N, device="cuda", dtype=torch.float32)
    g.gemm(a, b, acc, M, N, K, a_mn=a_mn, b_mn=b_mn, out_mode=1, splits=3)
    assert _rel(acc, A.float() @ B.float().t()) < 3e-3
    # split-K sums in a fixed order: bit-identical on repetition
    acc2 = torch.zeros_like(acc)
    g.gemm(a, b, acc2, M, N, K, a_mn=a_mn, b_mn=b_mn, out_mode=1, splits=3)
    assert torch.equal(acc, acc2)


def test_qkv_attention_matches_reference():
    from distributed_torch_horovod_gcp_b200.ops import functional as F2
    torch.manual_seed(12)
    B, S, D, H = 4, 197, 768, 12
    x = (torch.randn(B, S, D, device="cuda") * 0.5).to(torch.bfloat16).requires_grad_(True)
    w = (torch.randn(3 * D, D, device="cuda") * 0.03).to(torch.bfloat16).requires_grad_(True)
    b = (torch.randn(3 * D, device="cuda") * 0.1).to(torch.bfloat16).requires_grad_(True)
    xr, wr, br = [t.detach().float().requires_grad_(True) for t in (x, w, b)]
    y = F2.qkv_attention(x, w, b, H)
    yr = F2.attention_reference(torch.nn.functional.linear(xr, wr, br), H)
    assert y.shape == yr.shape and _rel(y, yr) < 2e-2
    g = torch.randn_like(y)
    y.backward(g)
    yr.backward(g.float())
    assert _rel(x.grad, xr.grad) < 3e-2
    assert _rel(w.grad, wr.grad) < 3e-2
    assert _rel(b.grad, br.grad) < 3e-2
