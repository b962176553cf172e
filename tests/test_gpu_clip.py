"""Clip by global norm inside the fused engine (``DistributedOptimizer(max_grad_norm=)``): one-shot reduce into
an fp32 arena + per-CTA norm slots, one finalize launch, one update launch per bucket."""
import copy
import os
import subprocess
import sys

import pytest
import torch
import torch.nn.functional as F

from mp_util import run_workers

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = torch.device("cuda", 0)


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


def _mlp():
    return torch.nn.Sequential(torch.nn.Linear(32, 100), torch.nn.ReLU(), torch.nn.Linear(100, 7)).to(DEV)


def _mk(opt_name, params):
    if opt_name == "sgd":
        return torch.optim.SGD(params, lr=0.1, momentum=0.9, weight_decay=1e-2, nesterov=True)
    if opt_name == "adam":
        return torch.optim.Adam(params, lr=1e-2)
    return torch.optim.AdamW(params, lr=1e-2, weight_decay=0.1)


def _launches_per_step(opt):
    """Clip mode: one reduce launch per bucket from the hooks, one finalize launch, one update per bucket."""
    return 2 * len(opt.bucket_plan()) + 1


def _against_torch(hvd, opt_name, dtype, bucket_bytes=None, steps=5, max_norm=0.02):
    torch.manual_seed(0)
    ref = _mlp()
    model = copy.deepcopy(ref).to(dtype)
    shadow = copy.deepcopy(ref).to(dtype)     # same bits as `model` every step -> the gradients the engine sees
    opt = hvd.DistributedOptimizer(_mk(opt_name, model.parameters()), named_parameters=model.named_parameters(),
                                   bucket_bytes=bucket_bytes, max_grad_norm=max_norm)
    assert opt.fused_engine is not None and opt.fused_engine.clip
    ropt = _mk(opt_name, ref.parameters())
    norm_t = opt.grad_norm
    x, y = torch.randn(16, 32, device=DEV), torch.randn(16, 7, device=DEV)
    for _ in range(steps):
        with torch.no_grad():
            for q, p in zip(shadow.parameters(), model.parameters()):
                q.copy_(p)
        shadow.zero_grad()
        F.mse_loss(shadow(x.to(dtype)).float(), y).backward()
        for p, q in zip(ref.parameters(), shadow.parameters()):
            p.grad = q.grad.float()
        exact = torch.linalg.vector_norm(torch.cat([p.grad.double().flatten() for p in ref.parameters()]))
        torch.nn.utils.clip_grad_norm_(ref.parameters(), max_norm)
        ropt.step()
        ropt.zero_grad()
        F.mse_loss(model(x.to(dtype)).float(), y).backward()
        opt.step()
        opt.zero_grad()
        assert opt.grad_norm is norm_t
        got = float(norm_t)
        assert got > max_norm, "max_norm must be small enough that every step clips"
        assert abs(got - float(exact)) <= 1e-5 * float(exact), (got, float(exact))
    tol = dict(rtol=1e-4, atol=1e-5) if dtype == torch.float32 else dict(rtol=2e-2, atol=2e-2)
    for a, b in zip(model.parameters(), ref.parameters()):
        torch.testing.assert_close(a.float(), b, **tol)
    assert opt.fused_engine.kernel_launches == steps * _launches_per_step(opt)
    return opt


@pytest.mark.parametrize("opt_name", ["sgd", "adam", "adamw"])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_clip_matches_torch(hvd1, opt_name, dtype):
    _against_torch(hvd1, opt_name, dtype)


def test_clip_norm_is_global_across_buckets(hvd1):
    opt = _against_torch(hvd1, "adamw", torch.float32, bucket_bytes=1024)
    assert len(opt.bucket_plan()) >= 3


def _engine_state(opt):
    out = []
    for ar in opt.fused_engine.arenas.values():
        out += [ar[k].clone() for k in ("M", "S0", "S1") if ar[k] is not None]
    return out + [opt.fused_engine.step_ctr.clone()]


def _run_fused(hvd, build, mk_opt, batches, max_grad_norm, steps=5):
    torch.manual_seed(0)
    model = build()
    opt = hvd.DistributedOptimizer(mk_opt(model.parameters()), named_parameters=model.named_parameters(),
                                   max_grad_norm=max_grad_norm)
    assert opt.fused_engine is not None
    norms = []
    for i in range(steps):
        x, y, loss_fn = batches[i % len(batches)]
        loss_fn(model(x), y).backward()
        opt.step()
        opt.zero_grad()
        if opt.grad_norm is not None:
            norms.append(opt.grad_norm.clone())
    torch.cuda.synchronize()
    params = [p.detach().clone() for p in model.parameters()]
    return params, _engine_state(opt), norms, opt


def _mlp_batches():
    torch.manual_seed(1)
    mse = lambda out, y: F.mse_loss(out.float(), y)
    return [(torch.randn(16, 32, device=DEV), torch.randn(16, 7, device=DEV), mse) for _ in range(3)]


def _resnet_build():
    from distributed_torch_horovod_gcp_b200.models import resnet50
    return resnet50(num_classes=10).to(DEV).to(torch.bfloat16).to(memory_format=torch.channels_last)


def _resnet_batches():
    torch.manual_seed(1)
    ce = lambda out, y: F.cross_entropy(out.float(), y)
    return [(torch.randn(8, 3, 64, 64, device=DEV, dtype=torch.bfloat16).contiguous(
        memory_format=torch.channels_last), torch.randint(0, 10, (8,), device=DEV), ce) for _ in range(2)]


@pytest.mark.parametrize("which", ["mlp", "resnet50_bf16"])
def test_noop_clip_is_bit_identical(hvd1, which):
    """max_grad_norm=1e30 clamps the coefficient to 1: (sum*scale)*1 through the same epilogue == the
    unclipped one-shot update, bit for bit (parameters, fp32 masters, optimizer state, step counters)."""
    if which == "mlp":
        build, batches = _mlp, _mlp_batches()
        mk_opt = lambda ps: _mk("adam", ps)
    else:
        build, batches = _resnet_build, _resnet_batches()
        mk_opt = lambda ps: torch.optim.SGD(ps, lr=0.05, momentum=0.9, weight_decay=1e-4)
    p0, s0, _, o0 = _run_fused(hvd1, build, mk_opt, batches, None)
    p1, s1, norms, o1 = _run_fused(hvd1, build, mk_opt, batches, 1e30)
    assert o0.fused_engine.clip is False and o1.fused_engine.clip is True
    assert all(0.0 < float(n) < 1e30 for n in norms)
    for a, b in zip(p0 + s0, p1 + s1):
        assert torch.equal(a, b)


def test_clip_runs_are_reproducible(hvd1):
    mk_opt = lambda ps: _mk("adamw", ps)
    build = lambda: _mlp().to(torch.bfloat16)
    batches = [(x.to(torch.bfloat16), y, l) for x, y, l in _mlp_batches()]
    p0, s0, n0, _ = _run_fused(hvd1, build, mk_opt, batches, 0.05)
    p1, s1, n1, _ = _run_fused(hvd1, build, mk_opt, batches, 0.05)
    assert all(float(n) > 0.05 for n in n0)
    for a, b in zip(p0 + s0 + n0, p1 + s1 + n1):
        assert torch.equal(a, b)


def test_clip_graph_replay_matches_eager(hvd1):
    """Whole-step CUDA graph with clip mode == eager; grad_norm is rewritten by every replay."""
    from distributed_torch_horovod_gcp_b200.utils.graph import GraphedStep
    hvd = hvd1
    torch.manual_seed(0)
    base = torch.nn.Sequential(torch.nn.Linear(64, 128), torch.nn.ReLU(), torch.nn.Linear(128, 8)).to(DEV)
    models = [copy.deepcopy(base) for _ in range(2)]
    opts = [hvd.DistributedOptimizer(torch.optim.SGD(m.parameters(), lr=0.05, momentum=0.9),
                                     named_parameters=m.named_parameters(), max_grad_norm=0.05) for m in models]
    assert all(o.fused_engine is not None and o.fused_engine.clip for o in opts)

    def make_step(m, o):
        def step(x, y):
            loss = F.mse_loss(m(x), y)
            loss.backward()
            o.step()
            o.zero_grad()
            return loss.detach()
        return step

    xs = [torch.randn(16, 64, device=DEV) for _ in range(6)]
    ys = [torch.randn(16, 8, device=DEV) for _ in range(6)]
    eager = make_step(models[0], opts[0])
    graphed = GraphedStep(make_step(models[1], opts[1]), [xs[0], ys[0]], warmup=2)
    assert graphed.kernels_per_replay >= _launches_per_step(opts[1])
    # bring the eager replica to the graphed one's state after its warm-up steps
    with torch.no_grad():
        for a, b in zip(models[0].parameters(), models[1].parameters()):
            a.copy_(b)
    opts[0].fused_engine.params_changed()
    for ar0, ar1 in zip(opts[0].fused_engine.arenas.values(), opts[1].fused_engine.arenas.values()):
        ar0["S0"].copy_(ar1["S0"])
    opts[0].fused_engine.step_ctr.copy_(opts[1].fused_engine.step_ctr)
    seen = []
    for x, y in zip(xs, ys):
        le = eager(x, y)
        lg = graphed(x, y)
        torch.testing.assert_close(le, lg, rtol=1e-5, atol=1e-6)
        torch.testing.assert_close(opts[1].grad_norm, opts[0].grad_norm, rtol=1e-5, atol=0.0)
        seen.append(float(opts[1].grad_norm))
    torch.cuda.synchronize()
    assert len(set(seen)) == len(seen), f"grad_norm was not updated by every replay: {seen}"
    assert all(v > 0.05 for v in seen)
    for a, b in zip(models[0].parameters(), models[1].parameters()):
        torch.testing.assert_close(a, b, rtol=1e-5, atol=1e-6)


@pytest.mark.parametrize("opt_name", ["sgd", "adam"])
def test_clip_checkpoint_resume(hvd1, opt_name, tmp_path):
    hvd = hvd1
    torch.manual_seed(0)

    def mk_model():
        return torch.nn.Sequential(torch.nn.Linear(32, 96), torch.nn.Tanh(), torch.nn.Linear(96, 5)).to(DEV)

    def mk_opt(m):
        base = torch.optim.SGD(m.parameters(), lr=0.05, momentum=0.9, weight_decay=1e-3) \
            if opt_name == "sgd" else torch.optim.Adam(m.parameters(), lr=1e-2)
        return hvd.DistributedOptimizer(base, named_parameters=m.named_parameters(), max_grad_norm=0.02)

    data = [(torch.randn(8, 32, device=DEV), torch.randn(8, 5, device=DEV)) for _ in range(6)]

    def run(m, o, batches):
        out = []
        for x, y in batches:
            F.mse_loss(m(x), y).backward()
            o.step()
            o.zero_grad()
            out.append(o.grad_norm.clone())
        return out

    m1 = mk_model()
    o1 = mk_opt(m1)
    assert o1.fused_engine is not None and o1.fused_engine.clip
    run(m1, o1, data[:3])
    ckpt = tmp_path / "ckpt.pt"
    torch.save({"model": m1.state_dict(), "opt": o1.state_dict()}, ckpt)
    n1 = run(m1, o1, data[3:])

    m2 = mk_model()
    o2 = mk_opt(m2)
    blob = torch.load(ckpt)
    m2.load_state_dict(blob["model"])
    hvd.broadcast_parameters(m2.state_dict(), root_rank=0)
    o2.load_state_dict(blob["opt"])
    n2 = run(m2, o2, data[3:])
    for a, b in zip(m1.parameters(), m2.parameters()):
        torch.testing.assert_close(a, b, rtol=1e-5, atol=1e-6)
    for a, b in zip(n1, n2):
        torch.testing.assert_close(a, b, rtol=1e-5, atol=0.0)
        assert float(a) > 0.02


def test_clip_step_without_backward_and_launch_count(hvd1):
    """step() with no backward reduces zero gradients: norm 0, coefficient clamped to 1, ordinary update
    (weight decay only).  kernel_launches == steps * (2 * buckets + 1)."""
    torch.manual_seed(0)
    m = _mlp()
    ref = copy.deepcopy(m)
    opt = hvd1.DistributedOptimizer(torch.optim.SGD(m.parameters(), lr=0.1, weight_decay=0.1),
                                    named_parameters=m.named_parameters(), bucket_bytes=1024, max_grad_norm=1.0)
    ropt = torch.optim.SGD(ref.parameters(), lr=0.1, weight_decay=0.1)
    nb = len(opt.bucket_plan())
    assert nb >= 3
    opt.step()
    for p in ref.parameters():
        p.grad = torch.zeros_like(p)
    ropt.step()
    torch.cuda.synchronize()
    assert float(opt.grad_norm) == 0.0
    for a, b in zip(m.parameters(), ref.parameters()):
        torch.testing.assert_close(a, b, rtol=1e-6, atol=1e-7)
    x, y = torch.randn(16, 32, device=DEV), torch.randn(16, 7, device=DEV)
    for _ in range(3):
        F.mse_loss(m(x), y).backward()
        opt.step()
        opt.zero_grad()
    assert opt.fused_engine.kernel_launches == 4 * (2 * nb + 1)


def test_skip_synchronize_error_points_to_max_grad_norm(hvd1):
    m = _mlp()
    opt = hvd1.DistributedOptimizer(torch.optim.SGD(m.parameters(), lr=0.1), named_parameters=m.named_parameters())
    assert opt.fused_engine is not None and opt.grad_norm is None
    F.mse_loss(m(torch.randn(4, 32, device=DEV)), torch.randn(4, 7, device=DEV)).backward()
    opt.synchronize()
    with pytest.raises(RuntimeError, match="max_grad_norm="):
        with opt.skip_synchronize():
            opt.step()


@pytest.mark.parametrize("graph", [False, True])
def test_app_script_clip_grad_norm(tmp_path, graph):
    env = dict(os.environ, PYTHONPATH=ROOT, B200DP_OFFLINE="1", B200DP_SYNTH_ROWS="2000")
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK", "B200DP_FUSED_SINGLE"):
        env.pop(k, None)
    cmd = [sys.executable, os.path.join(ROOT, "app", "torch_train.py"), "--epochs", "2", "--clip-grad-norm", "1.0"]
    if graph:
        cmd.append("--cuda-graph")
    r = subprocess.run(cmd, cwd=str(tmp_path), env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    assert "this process is using device - cuda:0" in r.stdout
    assert r.stdout.count("train_loss") == 2 and "total training time in minutes" in r.stdout
    assert "nan" not in r.stdout.split("train_loss")[-1]


def _world():
    n = torch.cuda.device_count()
    return 8 if n >= 8 else (4 if n >= 4 else 2)


@pytest.mark.multigpu
@pytest.mark.parametrize("opt_name", ["sgd", "adam"])
def test_multigpu_clip_matches_nccl(opt_name):
    res = run_workers(_world(), "clip_cases", "fused_clip_matches_nccl", (opt_name,), cuda=True, timeout=300)
    assert all(r[0] == res[0][0] for r in res), "grad_norm differs across ranks"
    assert len({r[1] for r in res}) == 1, "parameter digests differ across ranks"
