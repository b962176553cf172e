"""LARS / LAMB inside the fused engine: per bucket, a one-shot reduction that writes the update direction and
per-chunk partial norms (K10), then the trust ratios and the update (K11), both launched from the bucket's hook.
The eager ``hvd.LARS`` / ``hvd.LAMB`` ``step()`` is the reference."""
import copy
import hashlib
import os
import subprocess
import sys

import pytest
import torch
import torch.nn.functional as F

from fp64_bounds import assert_within_bound
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


class _Net(torch.nn.Module):
    """Several tensors of awkward sizes (biases of 7 and 3 elements end inside a 16-byte vector), plus a layer
    the loss never uses (its gradient stays zero; weight decay still moves it)."""

    def __init__(self):
        super().__init__()
        self.fc1, self.fc2, self.fc3 = torch.nn.Linear(32, 100), torch.nn.Linear(100, 64), torch.nn.Linear(64, 7)
        self.unused = torch.nn.Linear(5, 3)

    def forward(self, x):
        return self.fc3(F.relu(self.fc2(F.relu(self.fc1(x)))))


def _groups(model):
    named = list(model.named_parameters())
    return [{"params": [p for _, p in named if p.dim() > 1]},
            {"params": [p for _, p in named if p.dim() <= 1], "weight_decay": 0.0, "adaptive": False}]


def _mk(hvd, kind, params):
    if kind == "lars":
        return hvd.LARS(params, lr=0.5, momentum=0.9, weight_decay=1e-2, trust_coefficient=0.02)
    return hvd.LAMB(params, lr=0.02, betas=(0.9, 0.99), eps=1e-6, weight_decay=0.1)


def _masters(opt):
    """name -> the fp32 master of each parameter (the parameter itself when it is fp32)."""
    from distributed_torch_horovod_gcp_b200.parallel.fused_engine import arena_view
    eng, out = opt.fused_engine, {}
    for b in eng.buckets:
        ar = eng.arenas[b.dtype]
        src = ar["M"] if ar["M"] is not None else ar["p"]
        for s in b.slots:
            out[s.name] = arena_view(src, b.flat_offset + s.offset, s.param)
    return out


def _ratio64(kind, group, w, d):
    """The trust ratio in float64 from the master weight and the direction."""
    wn, dn = float(w.norm()), float(d.norm())
    coef = group["trust_coefficient"] if kind == "lars" else 1.0
    return coef * wn / dn if group["adaptive"] and wn > 0 and dn > 0 else 1.0


def _against_eager(hvd, kind, dtype, steps=5, bucket_bytes=1024, check_ratios=False):
    torch.manual_seed(0)
    model = _Net().to(DEV).to(dtype)
    ref = copy.deepcopy(model).float()           # fp32 eager reference of the masters, same starting values
    shadow = copy.deepcopy(model)                # same bits as `model` every step -> the gradients the engine sees
    opt = hvd.DistributedOptimizer(_mk(hvd, kind, _groups(model)), named_parameters=model.named_parameters(),
                                   bucket_bytes=bucket_bytes)
    eng = opt.fused_engine
    assert eng is not None and eng.layerwise and set(eng.algorithms().values()) == {"oneshot"}
    nb = len(opt.bucket_plan())
    assert nb >= 3
    ropt = _mk(hvd, kind, _groups(ref))
    group_of = {n: g for n, p in model.named_parameters() for g in opt.param_groups if any(p is q for q in g["params"])}
    x, y = torch.randn(16, 32, device=DEV), torch.randn(16, 7, device=DEV)
    for step in range(steps):
        with torch.no_grad():
            for q, p in zip(shadow.parameters(), model.parameters()):
                q.copy_(p)
        shadow.zero_grad()
        F.mse_loss(shadow(x.to(dtype)).float(), y).backward()
        grads = {n: (q.grad.float() if q.grad is not None else torch.zeros_like(q, dtype=torch.float32))
                 for n, q in shadow.named_parameters()}
        for (n, p) in ref.named_parameters():
            p.grad = grads[n].clone()
        w_before = {n: m.double().clone() for n, m in _masters(opt).items()}
        ropt.step()
        F.mse_loss(model(x.to(dtype)).float(), y).backward()
        opt.step()
        opt.zero_grad()
        if check_ratios and step == 0:
            _check_ratios(kind, eng, group_of, w_before, grads)
    tol = dict(rtol=1e-5, atol=1e-6) if dtype == torch.float32 else dict(rtol=1e-4, atol=1e-5)
    got = _masters(opt)
    for n, p in ref.named_parameters():
        torch.testing.assert_close(got[n].float(), p.detach(), **tol, msg=lambda m: f"{n}: {m}")
        if dtype != torch.float32:
            assert torch.equal(dict(model.named_parameters())[n].detach(), got[n].to(dtype))
    assert eng.kernel_launches == steps * 2 * nb
    return opt


def _check_ratios(kind, eng, group_of, w_before, grads):
    """First step: each tensor's ratio against float64 norms of the same master weights and gradients.  The
    bound is that of the fp32 sums of squares: a per-thread sequential run of at most VN * ceil(chunk / (512 *
    VN)) terms, two 32-lane butterflies, plus a few roundings of the direction per element and of sqrt / divide."""
    from distributed_torch_horovod_gcp_b200.parallel.fused_engine import LW_CHUNK_ELEMS
    ratios = eng.trust_ratios()
    torch.cuda.synchronize()
    assert set(ratios) == set(grads)
    for n, r in ratios.items():
        grp = group_of[n]
        w, g = w_before[n], grads[n].double()
        if kind == "lars":
            d = g + grp["weight_decay"] * w
        else:                     # step 1: m^ = g, sqrt(v^) = |g|
            d = g / (g.abs() + grp["eps"]) + grp["weight_decay"] * w
        want = _ratio64(kind, grp, w, d)
        if not grp["adaptive"]:
            assert float(r) == 1.0
            continue
        n_terms = 4 * -(-min(w.numel(), LW_CHUNK_ELEMS) // 2048) + 10 + 8
        want = torch.tensor([want], dtype=torch.float64)
        assert_within_bound(r.double().cpu().reshape(1), want, mag64=want, n_terms=n_terms,
                            group=f"trust ratio {kind}")


@pytest.mark.parametrize("kind", ["lars", "lamb"])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_fused_matches_eager(hvd1, kind, dtype):
    _against_eager(hvd1, kind, dtype)


@pytest.mark.parametrize("kind", ["lars", "lamb"])
def test_trust_ratios_match_float64(hvd1, kind):
    opt = _against_eager(hvd1, kind, torch.float32, steps=1, check_ratios=True)
    ratios = opt.fused_engine.trust_ratios()
    assert float(ratios["unused.weight"]) != 1.0 and float(ratios["unused.bias"]) == 1.0


def test_large_tensor_spans_chunks(hvd1):
    """A tensor of several chunks (partials folded across CTAs) and a bucket of many tensors."""
    from distributed_torch_horovod_gcp_b200.parallel.fused_engine import LW_CHUNK_ELEMS
    torch.manual_seed(0)
    model = torch.nn.Sequential(torch.nn.Linear(512, 300), torch.nn.Tanh(), torch.nn.Linear(300, 10)).to(DEV)
    assert model[0].weight.numel() > 8 * LW_CHUNK_ELEMS
    ref = copy.deepcopy(model)
    opt = hvd1.DistributedOptimizer(_mk(hvd1, "lars", _groups(model)), named_parameters=model.named_parameters())
    ropt = _mk(hvd1, "lars", _groups(ref))
    for _ in range(3):
        x, y = torch.randn(32, 512, device=DEV), torch.randn(32, 10, device=DEV)
        F.mse_loss(ref(x), y).backward()
        ropt.step()
        ropt.zero_grad()
        F.mse_loss(model(x), y).backward()
        opt.step()
        opt.zero_grad()
    for a, b in zip(model.parameters(), ref.parameters()):
        torch.testing.assert_close(a, b, rtol=1e-5, atol=1e-6)


def _run(hvd, kind, dtype, steps=4):
    torch.manual_seed(0)
    model = _Net().to(DEV).to(dtype)
    opt = hvd.DistributedOptimizer(_mk(hvd, kind, _groups(model)), named_parameters=model.named_parameters(),
                                   bucket_bytes=1024)
    torch.manual_seed(1)
    for _ in range(steps):
        x, y = torch.randn(16, 32, device=DEV, dtype=dtype), torch.randn(16, 7, device=DEV)
        F.mse_loss(model(x).float(), y).backward()
        opt.step()
        opt.zero_grad()
    torch.cuda.synchronize()
    eng = opt.fused_engine
    out = [p.detach().clone() for p in model.parameters()]
    for ar in eng.arenas.values():
        out += [ar[k].clone() for k in ("M", "S0", "S1") if ar[k] is not None]
    return out + [eng.step_ctr.clone(), eng.lw_ratio.clone()]


@pytest.mark.parametrize("kind", ["lars", "lamb"])
def test_runs_are_reproducible(hvd1, kind):
    a, b = _run(hvd1, kind, torch.bfloat16), _run(hvd1, kind, torch.bfloat16)
    for x, y in zip(a, b):
        assert torch.equal(x, y)


def test_both_phases_launch_inside_backward(hvd1):
    """When the last bucket's hook fires, both phases of every earlier bucket have been launched."""
    torch.manual_seed(0)
    model = torch.nn.Sequential(torch.nn.Linear(32, 100), torch.nn.ReLU(), torch.nn.Linear(100, 64),
                                torch.nn.ReLU(), torch.nn.Linear(64, 7)).to(DEV)
    opt = hvd1.DistributedOptimizer(_mk(hvd1, "lamb", _groups(model)), named_parameters=model.named_parameters(),
                                    bucket_bytes=1024)
    eng = opt.fused_engine
    nb = len(opt.bucket_plan())
    seen = []
    launch = eng.launch

    def spy(b):
        seen.append(eng.kernel_launches)
        return launch(b)
    eng.launch = spy
    F.mse_loss(model(torch.randn(16, 32, device=DEV)), torch.randn(16, 7, device=DEV)).backward()
    assert seen == [2 * i for i in range(nb)], seen       # every bucket launched during backward
    assert eng.kernel_launches == 2 * nb
    opt.step()
    assert eng.kernel_launches == 2 * nb


def test_graph_replay_matches_eager_and_honours_lr_scale(hvd1):
    """Whole-step CUDA graph with LAMB == the same engine run eagerly; ``lr_scale`` is read on every replay (at
    scale 0 a LAMB step leaves the parameters as they are)."""
    from distributed_torch_horovod_gcp_b200.utils.graph import GraphedStep
    hvd = hvd1
    torch.manual_seed(0)
    base = torch.nn.Sequential(torch.nn.Linear(64, 128), torch.nn.ReLU(), torch.nn.Linear(128, 8)).to(DEV)
    models = [copy.deepcopy(base) for _ in range(2)]
    opts = [hvd.DistributedOptimizer(_mk(hvd, "lamb", _groups(m)), named_parameters=m.named_parameters(),
                                     bucket_bytes=4096) for m in models]
    scales = []
    for o in opts:
        assert o.fused_engine is not None and o.fused_engine.layerwise
        o.fused_engine.lr_scale = torch.ones((), device=DEV)
        scales.append(o.fused_engine.lr_scale)

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
    assert graphed.kernels_per_replay >= 2 * len(opts[1].bucket_plan())
    # bring the eager replica to the graphed one's state after its warm-up steps
    with torch.no_grad():
        for a, b in zip(models[0].parameters(), models[1].parameters()):
            a.copy_(b)
    opts[0].fused_engine.params_changed()
    for ar0, ar1 in zip(opts[0].fused_engine.arenas.values(), opts[1].fused_engine.arenas.values()):
        ar0["S0"].copy_(ar1["S0"])
        ar0["S1"].copy_(ar1["S1"])
    opts[0].fused_engine.step_ctr.copy_(opts[1].fused_engine.step_ctr)
    for i, (x, y) in enumerate(zip(xs, ys)):
        for s in scales:
            s.fill_({3: 0.0, 4: 0.5}.get(i, 1.0))
        before = [p.detach().clone() for p in models[1].parameters()]
        le, lg = eager(x, y), graphed(x, y)
        torch.testing.assert_close(le, lg, rtol=1e-5, atol=1e-6)
        for a, b in zip(models[0].parameters(), models[1].parameters()):
            torch.testing.assert_close(a, b, rtol=1e-5, atol=1e-6)
        frozen = all(torch.equal(p, q) for p, q in zip(models[1].parameters(), before))
        assert frozen == (i == 3), f"replay {i}: lr_scale was not honoured"


@pytest.mark.parametrize("kind", ["lars", "lamb"])
def test_state_dict_round_trip_fused_eager_fused(hvd1, kind):
    hvd = hvd1
    torch.manual_seed(0)
    data = [(torch.randn(16, 32, device=DEV), torch.randn(16, 7, device=DEV)) for _ in range(7)]

    def fused_pair():
        m = _Net().to(DEV)
        return m, hvd.DistributedOptimizer(_mk(hvd, kind, _groups(m)), named_parameters=m.named_parameters(),
                                           bucket_bytes=1024)

    def run(m, o, batches):
        for x, y in batches:
            F.mse_loss(m(x), y).backward()
            if not hasattr(o, "fused_engine"):     # the eager optimizer sees the zero gradient the engine reduces
                for p in m.parameters():
                    if p.grad is None:
                        p.grad = torch.zeros_like(p)
            o.step()
            o.zero_grad(set_to_none=False)

    torch.manual_seed(1)
    m1, o1 = fused_pair()
    init = copy.deepcopy(m1.state_dict())
    run(m1, o1, data[:3])
    sd_model, sd_opt = copy.deepcopy(m1.state_dict()), copy.deepcopy(o1.state_dict())
    run(m1, o1, data[3:])                                   # the uninterrupted fused run

    m2 = _Net().to(DEV)
    m2.load_state_dict(sd_model)
    o2 = _mk(hvd, kind, _groups(m2))
    o2.load_state_dict(sd_opt)
    run(m2, o2, data[3:5])                                  # eager, from the fused checkpoint

    torch.manual_seed(1)
    m3, o3 = fused_pair()
    assert all(torch.equal(a, b) for a, b in zip(m3.state_dict().values(), init.values()))
    with torch.no_grad():
        for p, q in zip(m3.parameters(), m2.parameters()):
            p.copy_(q)
    o3.fused_engine.params_changed()
    o3.load_state_dict(copy.deepcopy(o2.state_dict()))     # fused, from the eager checkpoint
    run(m3, o3, data[5:])
    for a, b in zip(m1.parameters(), m3.parameters()):
        torch.testing.assert_close(a, b, rtol=1e-5, atol=1e-6)
    st = o3.state_dict()["state"]
    keys = {"lars": {"momentum_buffer"}, "lamb": {"step", "exp_avg", "exp_avg_sq"}}[kind]
    assert all(set(v) == keys for v in st.values())
    if kind == "lamb":
        assert all(float(v["step"]) == 7 for v in st.values())


def test_resnet18_bf16_lars_matches_generic_path(hvd1):
    from distributed_torch_horovod_gcp_b200.models import build
    hvd = hvd1
    torch.manual_seed(0)
    base = build("resnet18", num_classes=10, small_input=True).to(DEV).to(torch.bfloat16)
    base = base.to(memory_format=torch.channels_last).train()
    fused_m, generic_m = copy.deepcopy(base), copy.deepcopy(base)

    def mk(m):
        return hvd.LARS(_groups(m), lr=0.5, momentum=0.9, weight_decay=1e-4, trust_coefficient=0.02)

    fused = hvd.DistributedOptimizer(mk(fused_m), named_parameters=fused_m.named_parameters())
    generic = hvd.DistributedOptimizer(mk(generic_m), named_parameters=generic_m.named_parameters(), fused=False)
    assert fused.fused_engine is not None and fused.fused_engine.layerwise and generic.fused_engine is None
    torch.manual_seed(1)
    x = torch.randn(8, 3, 32, 32, device=DEV, dtype=torch.bfloat16).contiguous(memory_format=torch.channels_last)
    y = torch.randint(0, 10, (8,), device=DEV)
    for m, o in ((fused_m, fused), (generic_m, generic)):
        F.cross_entropy(m(x).float(), y).backward()
        o.step()
        o.zero_grad()
    torch.cuda.synchronize()
    moved = 0.0
    for (n, a), b, c in zip(fused_m.named_parameters(), generic_m.parameters(), base.parameters()):
        torch.testing.assert_close(a.float(), b.float(), rtol=2e-2, atol=2e-2, msg=lambda s: f"{n}: {s}")
        moved += float((a.detach().float() - c.detach().float()).abs().sum())
    assert moved > 0.0


def test_clip_or_compression_fall_back_to_generic_path(hvd1):
    torch.manual_seed(0)
    m = _Net().to(DEV)
    opt = hvd1.DistributedOptimizer(_mk(hvd1, "lars", _groups(m)), named_parameters=m.named_parameters(),
                                    max_grad_norm=1.0)
    assert opt.fused_engine is None
    F.mse_loss(m(torch.randn(4, 32, device=DEV)), torch.randn(4, 7, device=DEV)).backward()
    opt.step()
    assert 0.0 < float(opt.grad_norm) < float("inf")


def test_app_script_lars_cuda_graph(tmp_path):
    env = dict(os.environ, PYTHONPATH=ROOT, B200DP_OFFLINE="1")
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK", "B200DP_FUSED_SINGLE"):
        env.pop(k, None)
    cmd = [sys.executable, os.path.join(ROOT, "app", "torch_train.py"), "--model", "resnet18", "--dtype", "bf16",
           "--image-size", "32", "--num-classes", "10", "--batch-size", "16", "--epochs", "2",
           "--steps-per-epoch", "4", "--optimizer", "lars", "--cuda-graph"]
    r = subprocess.run(cmd, cwd=str(tmp_path), env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    losses = [float(s.split()[0].strip(",")) for s in r.stdout.split("train_loss: ")[1:]]
    assert len(losses) == 2 and all(v == v and abs(v) < float("inf") for v in losses), r.stdout


def _world():
    n = torch.cuda.device_count()
    return 8 if n >= 8 else (4 if n >= 4 else 2)


def fused_matches_nccl(hvd, kind):
    """Identical local gradients on both arms: (a) NCCL all_reduce average + the eager optimizer on a plain
    clone, (b) the fused engine.  Returns a digest of the updated parameters for the cross-rank comparison."""
    import torch.distributed as dist
    from distributed_torch_horovod_gcp_b200 import _state
    assert _state.get_symm() is not None, f"symmetric runtime unavailable: {_state.runtime().symm_failed}"
    r, n = hvd.rank(), hvd.size()
    dev = torch.device("cuda", torch.cuda.current_device())
    torch.manual_seed(0)
    model = torch.nn.Sequential(torch.nn.Linear(64, 300), torch.nn.Tanh(), torch.nn.Linear(300, 257),
                                torch.nn.Tanh(), torch.nn.Linear(257, 8)).to(dev)
    opt = hvd.DistributedOptimizer(_mk(hvd, kind, _groups(model)), named_parameters=model.named_parameters(),
                                   bucket_bytes=128 << 10)
    assert opt.fused_engine is not None and opt.fused_engine.layerwise
    hvd.broadcast_parameters(model.state_dict(), root_rank=0)
    ref = copy.deepcopy(model)
    for p in ref.parameters():
        p.grad = None
        if hasattr(p, "_b200dp_sink"):
            del p._b200dp_sink
    ropt = _mk(hvd, kind, _groups(ref))
    for step in range(3):
        torch.manual_seed(100 + 10 * step + r)
        x, y = torch.randn(16, 64, device=dev), torch.randn(16, 8, device=dev)
        for p in ref.parameters():
            p.grad = None
        F.mse_loss(ref(x), y).backward()
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
    for a, b in zip(model.parameters(), ref.parameters()):
        torch.testing.assert_close(a, b, rtol=2e-4, atol=2e-5)
    h = hashlib.sha256()
    for p in model.parameters():
        h.update(p.detach().contiguous().view(torch.uint8).cpu().numpy().tobytes())
    opt.remove_hooks()
    return h.hexdigest()


@pytest.mark.multigpu
@pytest.mark.parametrize("kind", ["lars", "lamb"])
def test_multigpu_matches_nccl_and_replicas_are_identical(kind):
    res = run_workers(_world(), "test_gpu_layerwise", "fused_matches_nccl", (kind,), cuda=True, timeout=300)
    assert len(set(res)) == 1, "parameter digests differ across ranks"
