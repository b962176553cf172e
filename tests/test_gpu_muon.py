"""Muon inside the fused engine: per Muon bucket, a one-shot reduction with the momentum update and per-chunk
sums of squares (K12), the per-matrix normalisation into bf16 (K13), the Newton–Schulz iterations on the wgmma
GEMM, and the update (K14), all launched from the bucket's hook; AdamW groups run K7.  The eager ``hvd.Muon``
``step()`` is the reference.  Also the GEMM's scaled residual, against float64 bounds."""
import copy
import ctypes
import logging

import numpy as np

import pytest
import torch
import torch.nn.functional as F

import launch_guard
from fp64_bounds import U32, assert_within_bound, report_ratios

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
NS_ABC = (3.4445, -4.775, 2.0315)
VN_OF = {torch.float32: 4, torch.bfloat16: 8}


@pytest.fixture
def hvd1(monkeypatch):
    """Single-process runtime with the fused engine at world size 1."""
    monkeypatch.setenv("B200DP_FUSED_SINGLE", "1")
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK", "LOCAL_WORLD_SIZE", "HOROVOD_TIMELINE"):
        monkeypatch.delenv(k, raising=False)
    import distributed_torch_horovod_gcp_b200.torch as hvd
    hvd.shutdown()
    hvd.init()
    yield hvd
    hvd.shutdown()


def teardown_module(module):
    report_ratios()


# ------------------------------------------------------------------------------------------ GEMM scaled residual
def _gemm64_bound(out, a, b, res, alpha, beta, K, group):
    a64, b64, r64 = a.double(), b.double(), res.double()
    ref = alpha * (a64 @ b64) + beta * r64
    mag = abs(alpha) * (a64.abs() @ b64.abs()) + abs(beta) * r64.abs()
    assert_within_bound(out, ref, mag, n_terms=K + 2, out_bf16=True, group=group)


@pytest.mark.parametrize("M,N,K", [(200, 264, 136), (768, 768, 768), (72, 1000, 520)])
@pytest.mark.parametrize("b_mn", [False, True])
@pytest.mark.parametrize("alpha,beta", [(2.0315, -4.775), (1.0, 3.4445), (1.0, 1.0)])
def test_gemm_scaled_residual_fp64_bound(M, N, K, b_mn, alpha, beta):
    from distributed_torch_horovod_gcp_b200.ops import gemm as G, kernels
    assert kernels.has("gemm")
    torch.manual_seed(M + N + K)
    a = torch.randn(M, K, device=DEV).bfloat16()
    bt = torch.randn(K, N, device=DEV).bfloat16()               # the math operand, [K, N]
    b = bt if b_mn else bt.t().contiguous()
    res = torch.randn(M, N, device=DEV).bfloat16()
    out = torch.empty(M, N, device=DEV, dtype=torch.bfloat16)
    G.gemm(a, b, out, M, N, K, b_mn=b_mn, residual=res, alpha=alpha, beta=beta)
    torch.cuda.synchronize()
    _gemm64_bound(out, a, bt, res, alpha, beta, K, "gemm scaled residual")


@pytest.mark.parametrize("M,N,K", [(200, 264, 136), (768, 768, 768)])
@pytest.mark.parametrize("b_mn", [False, True])
@pytest.mark.parametrize("alpha", [1.0, 2.0315])
def test_gemm_scaled_entry_at_beta_one_matches_unscaled_bits(M, N, K, b_mn, alpha):
    """b200dp_gemm_bf16_scaled called directly with beta = 1 (res_scale = 1 in the fma of the generic epilogue,
    and the res_only fast path when alpha = 1) gives the bits of b200dp_gemm_bf16."""
    from distributed_torch_horovod_gcp_b200.ops import gemm as G
    torch.manual_seed(M + N + K + 1)
    a = torch.randn(M, K, device=DEV).bfloat16()
    b = torch.randn(K, N, device=DEV).bfloat16() if b_mn else torch.randn(N, K, device=DEV).bfloat16()
    res = torch.randn(M, N, device=DEV).bfloat16()
    ref = torch.empty(M, N, device=DEV, dtype=torch.bfloat16)
    G.gemm(a, b, ref, M, N, K, b_mn=b_mn, residual=res, alpha=alpha)       # beta == 1: the unscaled entry point
    out = torch.full_like(ref, float("nan"))
    rc = G._lib.b200dp_gemm_bf16_scaled(
        a.data_ptr(), b.data_ptr(), out.data_ptr(), M, N, K, a.stride(0), b.stride(0), out.stride(0), 0, int(b_mn),
        None, None, res.data_ptr(), None, 0, 0, 1, alpha, 1.0, 1, 0, 0, None, None,
        torch.cuda.current_stream().cuda_stream)
    assert rc == 0, G._lib.b200dp_gemm_last_error()
    torch.cuda.synchronize()
    assert torch.equal(out, ref)


def test_gemm_scaled_residual_refuses_other_epilogues():
    from distributed_torch_horovod_gcp_b200.ops import gemm as G
    a = torch.randn(64, 64, device=DEV).bfloat16()
    out = torch.empty_like(a)
    with pytest.raises(RuntimeError, match="beta"):
        G.gemm(a, a, out, 64, 64, 64, beta=2.0)                          # no residual
    with pytest.raises(RuntimeError, match="beta"):
        G.gemm(a, a, out, 64, 64, 64, residual=a, act=3, beta=2.0)       # the residual is gelu's aux input


# ------------------------------------------------------------------------------------------ engine pieces
def _one_matrix(hvd, shape, ns_steps, dtype=torch.float32, grad=None, **kw):
    torch.manual_seed(0)
    w = torch.nn.Parameter(torch.randn(*shape, device=DEV, dtype=dtype) * 0.1)
    opt = hvd.DistributedOptimizer(hvd.Muon([w], lr=0.02, ns_steps=ns_steps, **kw), named_parameters=[("w", w)])
    eng = opt.fused_engine
    assert eng is not None and eng.muon
    g = grad if grad is not None else torch.randn(*shape, device=DEV)
    w0 = w.detach().float().clone()
    (w * g.to(dtype)).sum().backward()            # dL/dw = g
    opt.step()
    torch.cuda.synchronize()
    return w, w0, g.to(dtype).float(), eng


@pytest.mark.parametrize("shape", [(96, 200), (200, 96), (128, 128)])
def test_reduce_normalise_and_one_ns_stage_against_fp64(hvd1, shape):
    """ns_steps = 1 leaves X0 in ns_x[0], G and H of the one iteration in ns_g / ns_h and O in ns_x[1]: each
    stage is checked against float64 of the kernel's own inputs."""
    w, w0, g, eng = _one_matrix(hvd1, shape, ns_steps=1)
    mu = 0.95
    buf = torch.lerp(torch.zeros_like(g), g, 1 - mu)
    u = torch.lerp(g, buf, mu)
    ar = eng.arenas[torch.float32]
    n = g.numel()
    torch.testing.assert_close(ar["S0"][:n].view(shape), buf, rtol=0, atol=0)
    torch.testing.assert_close(ar["R"][:n].view(shape), u, rtol=0, atol=0)
    p, q = min(shape), max(shape)
    uw = u if shape[0] <= shape[1] else u.t()
    r = ar["R"][:n].view(shape).double()
    ref_x0 = (uw.double() / float(r.norm()))
    x0 = eng.ns_x[0][:n].view(p, q)
    assert_within_bound(x0, ref_x0, ref_x0.abs(), n_terms=4, out_bf16=True, group="muon X0")
    a, b, c = NS_ABC
    x64 = x0.double()
    gm = eng.ns_g[:p * p].view(p, p)
    assert_within_bound(gm, x64 @ x64.t(), x64.abs() @ x64.abs().t(), n_terms=q, out_bf16=True, group="muon G")
    g64 = gm.double()
    hm = eng.ns_h[:p * p].view(p, p)
    assert_within_bound(hm, c * (g64 @ g64) + b * g64, abs(c) * (g64.abs() @ g64.abs()) + abs(b) * g64.abs(),
                        n_terms=p + 2, out_bf16=True, group="muon H")
    h64 = hm.double()
    o = eng.ns_x[1][:n].view(p, q)
    assert_within_bound(o, a * x64 + h64 @ x64, abs(a) * x64.abs() + h64.abs() @ x64.abs(), n_terms=p + 2,
                        out_bf16=True, group="muon O")
    # the update from the kernel's own O, read back in the parameter's orientation
    o_w = (o if shape[0] <= shape[1] else o.t()).double()
    f = max(1.0, shape[0] / shape[1]) ** 0.5
    ref_w = w0.double() * (1 - 0.02 * 0.1) - 0.02 * f * o_w
    assert_within_bound(w.detach(), ref_w, w0.double().abs() + 0.02 * f * o_w.abs(), n_terms=3,
                        group="muon apply")


def test_ns_result_singular_values_in_the_quintic_band(hvd1):
    """Five iterations of the (3.4445, -4.775, 2.0315) quintic map every singular value of a full-rank matrix
    whose smallest one is not tiny into about [0.68, 1.13]; bf16 rounding widens that a little."""
    _, _, _, eng = _one_matrix(hvd1, (128, 384), ns_steps=5)
    o = eng.ns_x[1][:128 * 384].view(128, 384).double()
    s = torch.linalg.svdvals(o.cpu())
    assert float(s.min()) > 0.55 and float(s.max()) < 1.3, (float(s.min()), float(s.max()))


def test_zero_gradient_is_a_pure_weight_decay_step(hvd1):
    w, w0, _, eng = _one_matrix(hvd1, (64, 128), ns_steps=5, grad=torch.zeros(64, 128, device=DEV))
    decay = torch.tensor(1.0, dtype=torch.float32) - torch.tensor(0.02, dtype=torch.float32) * 0.1
    torch.testing.assert_close(w.detach(), w0 * decay.to(DEV), rtol=2 * U32, atol=0)
    assert torch.count_nonzero(eng.ns_x[0][:64 * 128]) == 0


# ------------------------------------------------------------------------------------------ whole engine vs eager
class _Net(torch.nn.Module):
    """A tall, a wide and a square matrix (the square one spans 16 chunks of 16384 elements), biases and an
    embedding in AdamW groups."""

    def __init__(self):
        super().__init__()
        self.emb = torch.nn.Embedding(40, 64)
        self.fc1, self.fc2 = torch.nn.Linear(64, 512), torch.nn.Linear(512, 512)
        self.fc3 = torch.nn.Linear(512, 64)

    def forward(self, t):
        return self.fc3(F.gelu(self.fc2(F.gelu(self.fc1(self.emb(t))))))


def _groups(model):
    named = list(model.named_parameters())
    return [{"params": [p for n, p in named if n.startswith("fc") and p.dim() == 2]},
            {"params": [p for n, p in named if n.startswith("emb")], "use_muon": False},
            {"params": [p for n, p in named if p.dim() < 2], "use_muon": False, "weight_decay": 0.0}]


def _mk(hvd, params, **kw):
    return hvd.Muon(params, lr=0.02, weight_decay=0.1, betas=(0.9, 0.95), **kw)


def _masters(opt):
    from distributed_torch_horovod_gcp_b200.parallel.fused_engine import arena_view
    eng, out = opt.fused_engine, {}
    for b in eng.buckets:
        ar = eng.arenas[b.dtype]
        src = ar["M"] if ar["M"] is not None else ar["p"]
        for s in b.slots:
            out[s.name] = arena_view(src, b.flat_offset + s.offset, s.param)
    return out


def _data(n=6, rows=1024):
    """Batches of ``rows`` tokens: more than every matrix's dimensions, so each gradient has full rank (NS maps
    every non-zero singular value towards 1, so directions a rank-deficient u barely holds would turn rounding
    noise into O(1) differences between two otherwise equal runs)."""
    torch.manual_seed(5)
    return [(torch.randint(0, 40, (rows,), device=DEV), torch.randn(rows, 64, device=DEV)) for _ in range(n)]


def _fused(hvd, dtype, bucket_bytes=1 << 20, **kw):
    torch.manual_seed(0)
    model = _Net().to(DEV).to(dtype)
    opt = hvd.DistributedOptimizer(_mk(hvd, _groups(model), **kw), named_parameters=model.named_parameters(),
                                   bucket_bytes=bucket_bytes)
    return model, opt


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_fused_matches_eager_muon(hvd1, dtype):
    """Gradients of the fused model feed an fp32 eager hvd.Muon, so both see the same inputs every step.  AdamW
    parameters and the momentum buffers must agree to fp32 rounding.  A Muon matrix's update is lr f O, and O is
    computed in bf16 by both (fused: the wgmma GEMM; eager: torch's matmuls), with different roundings that the
    quintic amplifies (a slope up to a = 3.4445 per iteration on small singular values): so at every step the
    fused O, recovered from the master weights, must be no further from a float64 Newton–Schulz of the kernel's own
    u than torch's bf16 Newton–Schulz of the same u is, up to a factor 2 (plus 1% of ‖O‖)."""
    from distributed_torch_horovod_gcp_b200.torch.optim import muon_lr_ratio, newton_schulz
    hvd = hvd1
    model, opt = _fused(hvd, dtype, bucket_bytes=64 << 10)
    eng = opt.fused_engine
    assert eng is not None and eng.muon and set(eng.algorithms().values()) == {"oneshot"}
    assert len(opt.bucket_plan()) >= 3 and len(eng._mu_args) >= 2
    ref = copy.deepcopy(model).float()
    shadow = copy.deepcopy(model)
    ropt = _mk(hvd, _groups(ref))
    muon_names = [n for n, p in ref.named_parameters() if n.startswith("fc") and p.dim() == 2]
    slots = {s.name: (b, s) for b in eng.buckets for s in b.slots}
    lr, wd = 0.02, 0.1
    for t, y in _data():
        with torch.no_grad():
            for q, p in zip(shadow.parameters(), model.parameters()):
                q.copy_(p)
        shadow.zero_grad()
        F.mse_loss(shadow(t).float(), y).backward()
        for (n, p), q in zip(ref.named_parameters(), shadow.parameters()):
            p.grad = q.grad.float().clone()
        ropt.step()
        before = {n: m.double().clone() for n, m in _masters(opt).items()}
        F.mse_loss(model(t).float(), y).backward()
        opt.step()
        opt.zero_grad()
        got = _masters(opt)
        for n in muon_names:
            b, s = slots[n]
            shape = s.param.shape
            u = eng.arenas[b.dtype]["R"][b.flat_offset + s.offset: b.flat_offset + s.offset + s.numel].view(shape)
            step = float(torch.tensor(lr, dtype=torch.float32)) * muon_lr_ratio(None, shape)
            o_fused = (before[n] * (1 - lr * wd) - got[n].double()) / step
            o_eager = newton_schulz(u, NS_ABC, 5, 1e-7).double()
            o64 = _ns64(u)
            e_f, e_e = float((o_fused - o64).norm()), float((o_eager - o64).norm())
            assert e_f <= 2 * e_e + 0.01 * float(o64.norm()), f"{n}: fused {e_f:.4g} vs torch bf16 {e_e:.4g}"
    got = _masters(opt)
    sd = opt.state_dict()["state"]                  # indexed in param-group order
    name_of = {id(p): n for n, p in ref.named_parameters()}
    for i, p in enumerate(q for g in ropt.param_groups for q in g["params"]):
        n = name_of[id(p)]
        if n in muon_names:
            torch.testing.assert_close(sd[i]["momentum_buffer"].float(), ropt.state[p]["momentum_buffer"],
                                       rtol=1e-4, atol=1e-6)
        else:
            torch.testing.assert_close(got[n].float(), p.detach(), rtol=1e-4, atol=1e-5, msg=lambda m: f"{n}: {m}")
        if dtype != torch.float32:
            assert torch.equal(dict(model.named_parameters())[n].detach(), got[n].to(dtype))


def _ns64(u):
    """The quintic Newton–Schulz iteration in float64 (no bf16 roundings)."""
    a, b, c = NS_ABC
    x = u.double()
    tall = x.shape[0] > x.shape[1]
    if tall:
        x = x.t()
    x = x / x.norm().clamp(min=1e-7)
    for _ in range(5):
        g = x @ x.t()
        x = a * x + (c * (g @ g) + b * g) @ x
    return x.t() if tall else x



def _run_fused(hvd, steps=4):
    model, opt = _fused(hvd, torch.bfloat16, bucket_bytes=64 << 10)
    for t, y in _data(steps):
        F.mse_loss(model(t).float(), y).backward()
        opt.step()
        opt.zero_grad()
    torch.cuda.synchronize()
    return [p.detach().clone() for p in model.parameters()]


def test_two_runs_are_bitwise_identical(hvd1):
    a, b = _run_fused(hvd1), _run_fused(hvd1)
    assert all(torch.equal(x, y) for x, y in zip(a, b))


def test_every_phase_is_launched_inside_backward(hvd1):
    model, opt = _fused(hvd1, torch.float32, bucket_bytes=64 << 10)
    eng = opt.fused_engine
    nb = len(opt.bucket_plan())
    t, y = _data(1)[0]
    F.mse_loss(model(t), y).backward()
    assert len(opt._launched) == nb                     # every bucket's hook fired during backward
    ns = sum(3 * 5 * len(eng._mu_mats[i]) for i in eng._mu_args)
    assert eng.kernel_launches == nb + 2 * len(eng._mu_args) + ns
    opt.step()
    assert eng.kernel_launches == nb + 2 * len(eng._mu_args) + ns   # step() launches nothing


def test_graph_replay_matches_eager_and_honours_lr_scale(hvd1):
    from distributed_torch_horovod_gcp_b200.utils.graph import GraphedStep
    hvd = hvd1
    pairs = [_fused(hvd, torch.float32, bucket_bytes=64 << 10) for _ in range(2)]
    models, opts = [m for m, _ in pairs], [o for _, o in pairs]
    scales = []
    for o in opts:
        o.fused_engine.lr_scale = torch.ones((), device=DEV)
        scales.append(o.fused_engine.lr_scale)

    def make_step(m, o):
        def step(t, y):
            loss = F.mse_loss(m(t), y)
            loss.backward()
            o.step()
            o.zero_grad()
            return loss.detach()
        return step

    data = _data(6)
    eager = make_step(models[0], opts[0])
    graphed = GraphedStep(make_step(models[1], opts[1]), list(data[0]), warmup=2)
    with torch.no_grad():
        for a, b in zip(models[0].parameters(), models[1].parameters()):
            a.copy_(b)
    e0, e1 = opts[0].fused_engine, opts[1].fused_engine
    e0.params_changed()
    for ar0, ar1 in zip(e0.arenas.values(), e1.arenas.values()):
        ar0["S0"].copy_(ar1["S0"])
        ar0["S1"].copy_(ar1["S1"])
    e0.step_ctr.copy_(e1.step_ctr)
    for i, (t, y) in enumerate(data):
        for s in scales:
            s.fill_({3: 0.0, 4: 0.5}.get(i, 1.0))
        before = [p.detach().clone() for p in models[1].parameters()]
        le, lg = eager(t, y), graphed(t, y)
        assert torch.equal(le, lg)
        for a, b in zip(models[0].parameters(), models[1].parameters()):
            assert torch.equal(a, b)
        frozen = all(torch.equal(p, q) for p, q in zip(models[1].parameters(), before))
        assert frozen == (i == 3), f"replay {i}: lr_scale was not honoured"


def test_state_dict_round_trip_fused_eager_fused(hvd1):
    """Fused state -> eager hvd.Muon -> fused again carries momentum buffers and AdamW moments exactly: the
    reloaded engine continues bit for bit like the engine that never stopped.  The eager optimizer also steps from
    the loaded state."""
    hvd = hvd1
    data = _data(6)

    def run(m, o, batches):
        for t, y in batches:
            F.mse_loss(m(t), y).backward()
            o.step()
            o.zero_grad(set_to_none=False)

    m1, o1 = _fused(hvd, torch.float32)
    run(m1, o1, data[:3])
    sd, wsd = copy.deepcopy(o1.state_dict()), copy.deepcopy(m1.state_dict())
    assert any("momentum_buffer" in st for st in sd["state"].values())
    assert any("exp_avg_sq" in st for st in sd["state"].values())
    m2 = _Net().to(DEV)
    m2.load_state_dict(wsd)
    o2 = _mk(hvd, _groups(m2))
    o2.load_state_dict(sd)
    sd2 = copy.deepcopy(o2.state_dict())
    m3, o3 = _fused(hvd, torch.float32)
    m3.load_state_dict(wsd)
    o3.load_state_dict(sd2)
    s1, s3 = o1.state_dict()["state"], o3.state_dict()["state"]
    for i in s1:
        for k in s1[i]:
            assert torch.equal(s1[i][k].float().cpu(), s3[i][k].float().cpu()), (i, k)
    run(m1, o1, data[3:])
    run(m3, o3, data[3:])
    for a, b in zip(m1.parameters(), m3.parameters()):
        assert torch.equal(a, b)
    before = [p.detach().clone() for p in m2.parameters()]
    run(m2, o2, data[3:4])
    assert all(torch.isfinite(p).all() and not torch.equal(p, q) for p, q in zip(m2.parameters(), before))


@pytest.mark.parametrize("how", ["clip", "compression"])
def test_clipping_and_compression_fall_back_with_one_log_line(hvd1, how, caplog):
    from distributed_torch_horovod_gcp_b200.parallel import fused_engine
    hvd = hvd1
    fused_engine._logged_layerwise_fallback = False
    kw = {"max_grad_norm": 1.0} if how == "clip" else {"compression": hvd.Compression.bf16}
    with caplog.at_level(logging.WARNING, logger="b200dp"):
        for _ in range(2):
            m = _Net().to(DEV)
            opt = hvd.DistributedOptimizer(_mk(hvd, _groups(m)), named_parameters=m.named_parameters(), **kw)
            assert opt.fused_engine is None
            t, y = _data(1)[0]
            F.mse_loss(m(t), y).backward()
            opt.step()
    lines = [r for r in caplog.records if "Muon" in r.getMessage() and "generic path" in r.getMessage()]
    assert len(lines) == 1


def test_engine_launches_pass_the_host_launch_guard(hvd1, monkeypatch):
    """The NS GEMMs' new entry point is described in the guard's table here: the scaled-residual form has the
    arguments of b200dp_gemm_bf16 plus beta."""
    names, ptrs = launch_guard.TABLE["b200dp_gemm_bf16"]
    i = names.index("alpha") + 1
    monkeypatch.setitem(launch_guard.TABLE, "b200dp_gemm_bf16_scaled", (names[:i] + ("beta",) + names[i:], ptrs))
    calls = launch_guard.install(monkeypatch)
    model, opt = _fused(hvd1, torch.bfloat16, bucket_bytes=64 << 10)
    for t, y in _data(2):
        F.mse_loss(model(t).float(), y).backward()
        opt.step()
        opt.zero_grad()
    torch.cuda.synchronize()
    eng = opt.fused_engine
    nmat = sum(len(eng._mu_mats[i]) for i in eng._mu_args)
    assert calls["b200dp_gemm_bf16_scaled"] == 2 * 2 * 5 * nmat
    assert calls["b200dp_gemm_bf16"] == 2 * 5 * nmat


def test_generic_path_when_a_matrix_is_not_a_multiple_of_8(hvd1, caplog):
    from distributed_torch_horovod_gcp_b200.parallel import fused_engine
    hvd = hvd1
    fused_engine._logged_muon_fallback = False
    w = torch.nn.Parameter(torch.randn(12, 20, device=DEV))
    with caplog.at_level(logging.WARNING, logger="b200dp"):
        opt = hvd.DistributedOptimizer(hvd.Muon([w]), named_parameters=[("w", w)])
    assert opt.fused_engine is None
    assert any("multiple of 8" in r.getMessage() for r in caplog.records)


# ------------------------------------------------------------------------------------------ K12 at world sizes 1-8
def _f32_fma(a, b, c):
    """fp32 fma(a, b, c) of fp32 CPU tensors: the product is exact in float64 and the sum rounds once there
    before the rounding to fp32 (a double rounding that the fixed inputs here never hit)."""
    return (a.double() * b.double() + c.double()).float()


def _lerp32(s, e, w):
    """torch.lerp's formula in fp32 with the fma the kernel uses, for a scalar weight w (an fp32 value)."""
    w32 = torch.tensor(w, dtype=torch.float32)
    d = e - s                                   # fp32 subtraction, rounded once
    if abs(w) < 0.5:
        return _f32_fma(w32.expand_as(d), d, s)
    return _f32_fma(-d, (torch.tensor(1.0, dtype=torch.float32) - w32).expand_as(d), e)


@pytest.mark.parametrize("N", [1, 2, 3, 4, 5, 6, 7, 8])
@pytest.mark.parametrize("dtype,grid,nesterov", [(torch.float32, 7, True), (torch.bfloat16, 128, False),
                                                 (torch.bfloat16, 1, True)])
def test_muon_reduction_at_emulated_world_sizes(N, dtype, grid, nesterov):
    """K12 as rank r of a world of N on one GPU (the emulation of test_gpu_comm_numerics): on every rank S0 and R
    equal, bit for bit, the rank-order fp32 sum times the fp32 scale 1/N pushed through the momentum lerp and
    the nesterov lerp; the per-chunk sums of squares are the same bits on every rank and within the float64 bound
    of the sum of u^2; each rank writes only its own S0, R and partials and zeroes only its own gradient, after
    the closing barrier; guard elements stay untouched."""
    from test_gpu_comm_numerics import CH_USER, DT_CODE, GUARD, THREADS, Emu, _buf, _stream, ar_args, owned_by, \
        rank_sum, same_values
    from test_gpu_optimizer_numerics import Checker, _lw_layout
    from distributed_torch_horovod_gcp_b200.runtime import symm as S
    n, tens, rows = _lw_layout(dtype, [64 * 800, 24 * 40, 16 * 16, 8 * 2048])
    nch = len(rows)
    assert nch > len(tens)                      # a matrix spans several chunks
    gen = torch.Generator().manual_seed(10 * N + grid)
    gs = [torch.randn(n, generator=gen).to(dtype) for _ in range(N)]
    buf0 = torch.randn(n, generator=gen) * 0.1
    mu = 0.95
    emu, ck = Emu(N, seed=n + N), Checker()
    chunks = torch.tensor(rows, dtype=torch.int32, device="cuda")
    p = torch.randn(n, generator=gen)
    inp = [_buf(n, dtype, g) for g in gs]
    out = [_buf(n, dtype, p.to(dtype)) for _ in range(N)]
    s0 = [_buf(n, torch.float32, buf0) for _ in range(N)]
    r32, part = [_buf(n, torch.float32) for _ in range(N)], [_buf(2 * nch, torch.float32) for _ in range(N)]

    def fn(r, ctx):
        a = ar_args(inp, out, n, 1.0 / N, CH_USER, 1)
        a.s0 = s0[r].data_ptr()
        a.h.kind, a.h.lr, a.h.momentum, a.h.dampening = S.OPT_MUON, 0.02, mu, float(1 - mu)
        k = S.MuonArgs()
        k.r, k.part, k.chunks, k.nchunks = r32[r].data_ptr(), part[r].data_ptr(), chunks.data_ptr(), nch
        k.nesterov, k.eps = int(nesterov), 1e-7
        return emu.lib.b200dp_comm_muon_bucket(ctypes.byref(ctx), ctypes.byref(a), ctypes.byref(k), S.MUON_REDUCE,
                                               DT_CODE[dtype], grid, THREADS, _stream())
    bufs = {"in": inp, "out": out, "s0": s0, "r": r32, "part": part}
    fin, owner = emu.isolated(ck, "K12", bufs, fn, CH_USER, grid)
    g = rank_sum(gs) * torch.tensor(float(np.float32(1.0 / N)), dtype=torch.float32)
    b_ref = _lerp32(buf0, g, float(np.float32(1 - mu)))
    u_ref = _lerp32(g, b_ref, float(np.float32(mu))) if nesterov else b_ref
    u64 = u_ref.double()
    for q in range(N):
        ck.true("K12 S0", same_values(fin["s0"][q][:n], b_ref), f"rank {q}")
        ck.true("K12 R", same_values(fin["r"][q][:n], u_ref), f"rank {q}")
        ck.same_bits("K12 partials agree", fin["part"][q][:2 * nch], fin["part"][0][:2 * nch])
        pq = fin["part"][q][:2 * nch].cpu().view(nch, 2)
        ck.true("K12 second partial", bool((pq[:, 1] == 0).all()), f"rank {q}")
        for c, (v0, nv, _, _) in enumerate(rows):
            seg = u64[v0 * VN_OF[dtype]: (v0 + nv) * VN_OF[dtype]]
            exact = float((seg * seg).sum())
            assert abs(float(pq[c, 0]) - exact) <= 2 * (seg.numel() + 1) * U32 * exact, (q, c)
        # every element of R and the partials is written (they start as a sentinel NaN) by rank q alone; S0 and
        # the gradient only by rank q; nothing past an end (the GUARD elements) and nothing in the parameters
        ck.true("K12 write set", owned_by(owner["r"][q], torch.full((n,), q, device="cuda")) and
                owned_by(owner["part"][q], torch.full((2 * nch,), q, device="cuda")) and
                bool((owner["out"][q] == -1).all()), f"rank {q}")
        for k in ("s0", "in"):
            ck.true("K12 guard", bool((owner[k][q][-GUARD:] == -1).all()), f"{k} of rank {q}")
            ck.true("K12 owner", bool(((owner[k][q][:n] == q) | (owner[k][q][:n] == -1)).all()), f"{k} of rank {q}")
        ck.same_bits("K12 zero_input", fin["in"][q][:n], torch.zeros(n, dtype=dtype, device="cuda"))
    ck.close()


# ------------------------------------------------------------------------------------------ 2+ GPUs
def _world():
    n = torch.cuda.device_count()
    return 8 if n >= 8 else (4 if n >= 4 else 2)


def fused_matches_generic(hvd):
    """Identical local gradients on both arms: (a) NCCL all_reduce average + the eager hvd.Muon on a plain clone
    (the generic path's arithmetic), (b) the fused engine.  AdamW parameters and momentum buffers agree to fp32
    rounding; each step's fused O, recovered from the masters, is no further from a float64 Newton–Schulz of the
    fused u than torch's bf16 Newton–Schulz of that u is, up to a factor 2 (plus 1% of |O|), as in the one-GPU
    test.  Returns a digest of the parameters for the cross-rank comparison."""
    import hashlib

    import torch.distributed as dist
    from distributed_torch_horovod_gcp_b200 import _state
    from distributed_torch_horovod_gcp_b200.torch.optim import muon_lr_ratio, newton_schulz
    assert _state.get_symm() is not None, f"symmetric runtime unavailable: {_state.runtime().symm_failed}"
    r, n = hvd.rank(), hvd.size()
    dev = torch.device("cuda", torch.cuda.current_device())
    torch.manual_seed(0)
    model = _Net().to(dev)
    opt = hvd.DistributedOptimizer(_mk(hvd, _groups(model)), named_parameters=model.named_parameters(),
                                   bucket_bytes=256 << 10)
    eng = opt.fused_engine
    assert eng is not None and eng.muon and len(eng._mu_args) >= 2
    hvd.broadcast_parameters(model.state_dict(), root_rank=0)
    ref = copy.deepcopy(model)
    for p in ref.parameters():
        p.grad = None
        if hasattr(p, "_b200dp_sink"):
            del p._b200dp_sink
    ropt = _mk(hvd, _groups(ref))
    muon = [name for name, p in model.named_parameters() if name.startswith("fc") and p.dim() == 2]
    slots = {s.name: (b, s) for b in eng.buckets for s in b.slots}
    for step in range(3):
        torch.manual_seed(100 + 10 * step + r)
        t, y = torch.randint(0, 40, (1024,), device=dev), torch.randn(1024, 64, device=dev)
        for p in ref.parameters():
            p.grad = None
        F.mse_loss(ref(t), y).backward()
        before = {k: m.double().clone() for k, m in _masters(opt).items()}
        with torch.no_grad():
            for p, q in zip(model.parameters(), ref.parameters()):
                p.grad.copy_(q.grad)
        opt.step()
        opt.zero_grad()
        for p in ref.parameters():
            dist.all_reduce(p.grad)
            p.grad /= n
        ropt.step()
        torch.cuda.synchronize()
        got = _masters(opt)
        for name in muon:
            b, s = slots[name]
            u = eng.arenas[b.dtype]["R"][b.flat_offset + s.offset: b.flat_offset + s.offset + s.numel].view(s.param.shape)
            stp = float(torch.tensor(0.02, dtype=torch.float32)) * muon_lr_ratio(None, s.param.shape)
            o_fused = (before[name] * (1 - 0.02 * 0.1) - got[name].double()) / stp
            o64 = _ns64(u)
            e_f = float((o_fused - o64).norm())
            e_e = float((newton_schulz(u, NS_ABC, 5, 1e-7).double() - o64).norm())
            assert e_f <= 2 * e_e + 0.01 * float(o64.norm()), f"{name}: fused {e_f:.4g} vs torch bf16 {e_e:.4g}"
    name_of = {id(p): k for k, p in ref.named_parameters()}
    sd = opt.state_dict()["state"]
    for i, p in enumerate(q for g in ropt.param_groups for q in g["params"]):
        if name_of[id(p)] in muon:
            torch.testing.assert_close(sd[i]["momentum_buffer"].float(), ropt.state[p]["momentum_buffer"],
                                       rtol=1e-4, atol=1e-6)
        else:
            torch.testing.assert_close(dict(model.named_parameters())[name_of[id(p)]], p, rtol=1e-4, atol=1e-5)
    h = hashlib.sha256()
    for p in model.parameters():
        h.update(p.detach().contiguous().view(torch.uint8).cpu().numpy().tobytes())
    opt.remove_hooks()
    return h.hexdigest()


@pytest.mark.multigpu
def test_multigpu_replicas_identical_and_fused_matches_generic():
    from mp_util import run_workers
    res = run_workers(_world(), "test_gpu_muon", "fused_matches_generic", (), cuda=True, timeout=300)
    assert len(set(res)) == 1, "parameter digests differ across ranks"
