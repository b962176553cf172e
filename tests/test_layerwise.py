"""``hvd.LARS`` / ``hvd.LAMB`` without a GPU: the eager update against a float64 transcription of the rules,
argument validation, the generic DistributedOptimizer path over Gloo and the training script's flag."""
import copy
import os
import subprocess
import sys

import pytest
import torch
import torch.nn.functional as F

from mp_util import run_workers

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _ref_step(kind, ws, gs, state, groups, t):
    """One step of the rules in float64.  ws / gs: lists of float64 tensors; groups: per tensor dict."""
    for i, (w, g, grp) in enumerate(zip(ws, gs, groups)):
        wd, lr = grp["weight_decay"], grp["lr"]
        if kind == "lars":
            d = g + wd * w
            coef = grp["trust_coefficient"]
        else:
            b1, b2 = grp["betas"]
            m, v = state.setdefault(i, (torch.zeros_like(w), torch.zeros_like(w)))
            m = b1 * m + (1 - b1) * g
            v = b2 * v + (1 - b2) * g * g
            state[i] = (m, v)
            d = (m / (1 - b1 ** t)) / (v.sqrt() / (1 - b2 ** t) ** 0.5 + grp["eps"]) + wd * w
            coef = 1.0
        wn, dn = float(w.norm()), float(d.norm())
        trust = coef * wn / dn if grp["adaptive"] and wn > 0 and dn > 0 else 1.0
        if kind == "lars":
            buf = grp["momentum"] * state.get(i, torch.zeros_like(w)) + lr * trust * d
            state[i] = buf
            w -= buf
        else:
            w -= lr * trust * d


def _case():
    """Mixed groups: an adaptive group with weight decay (holding an all-zero weight), a non-adaptive group
    without decay, and an adaptive group without decay holding a tensor whose gradient is always zero."""
    torch.manual_seed(0)
    ps = [torch.nn.Parameter(torch.randn(8, 5)), torch.nn.Parameter(torch.zeros(4, 3)),
          torch.nn.Parameter(torch.randn(8)), torch.nn.Parameter(torch.randn(3, 3)),
          torch.nn.Parameter(torch.randn(6, 2))]
    groups = [{"params": ps[0:2]}, {"params": [ps[2]], "weight_decay": 0.0, "adaptive": False},
              {"params": ps[3:5], "weight_decay": 0.0}]
    grads = [[torch.randn_like(p) for p in ps] for _ in range(5)]
    for g in grads:
        g[3].zero_()
    return ps, groups, grads


@pytest.mark.parametrize("kind", ["lars", "lamb"])
def test_eager_matches_float64_rules(kind):
    import distributed_torch_horovod_gcp_b200.torch as hvd
    ps, groups, grads = _case()
    if kind == "lars":
        opt = hvd.LARS(groups, lr=0.5, momentum=0.9, weight_decay=1e-2, trust_coefficient=0.02)
    else:
        opt = hvd.LAMB(groups, lr=0.05, betas=(0.8, 0.95), eps=1e-6, weight_decay=0.1)
    per_tensor = [g for g in opt.param_groups for _ in g["params"]]
    ws = [p.detach().double().clone() for p in ps]
    state = {}
    for t, gs in enumerate(grads, start=1):
        for p, g in zip(ps, gs):
            p.grad = g.clone()
        opt.step()
        _ref_step(kind, ws, [g.double() for g in gs], state, per_tensor, t)
        for p, w in zip(ps, ws):
            torch.testing.assert_close(p.detach().double(), w, rtol=2e-5, atol=1e-6)
    assert float(ps[1].detach().abs().sum()) > 0.0, "the zero weight must have moved (trust 1)"
    torch.testing.assert_close(ps[3].detach().double(), _case()[0][3].detach().double(), rtol=0, atol=0)
    keys = {"lars": {"momentum_buffer"}, "lamb": {"step", "exp_avg", "exp_avg_sq"}}[kind]
    assert all(set(opt.state[p]) == keys for p in ps)
    if kind == "lamb":
        assert float(opt.state[ps[0]]["step"]) == len(grads)


@pytest.mark.parametrize("kwargs", [dict(lr=-0.1), dict(momentum=-0.1), dict(momentum=1.0), dict(weight_decay=-1e-4),
                                    dict(trust_coefficient=-1.0), dict(maximize=True)])
def test_lars_rejects_bad_arguments(kwargs):
    import distributed_torch_horovod_gcp_b200.torch as hvd
    with pytest.raises(ValueError):
        hvd.LARS(torch.nn.Linear(2, 2).parameters(), **kwargs)


@pytest.mark.parametrize("kwargs", [dict(lr=-1e-3), dict(betas=(1.0, 0.999)), dict(betas=(0.9, -0.1)),
                                    dict(betas=(0.9, 1.0)), dict(eps=-1e-6), dict(weight_decay=-0.01),
                                    dict(maximize=True)])
def test_lamb_rejects_bad_arguments(kwargs):
    import distributed_torch_horovod_gcp_b200.torch as hvd
    with pytest.raises(ValueError):
        hvd.LAMB(torch.nn.Linear(2, 2).parameters(), **kwargs)


def test_bad_param_group_is_rejected():
    import distributed_torch_horovod_gcp_b200.torch as hvd
    m = torch.nn.Linear(2, 2)
    opt = hvd.LARS([m.weight])
    with pytest.raises(ValueError):
        opt.add_param_group({"params": [m.bias], "maximize": True})
    with pytest.raises(ValueError):
        hvd.LAMB([{"params": [m.weight]}, {"params": [m.bias], "lr": -1.0}])


def test_classified_for_the_fused_engine():
    import distributed_torch_horovod_gcp_b200.torch as hvd
    from distributed_torch_horovod_gcp_b200.parallel.fused_engine import _classify
    ps = list(torch.nn.Linear(2, 2).parameters())
    assert _classify(hvd.LARS(ps)) == "lars"
    assert _classify(hvd.LAMB(ps)) == "lamb"


def gloo_trains(hvd, kind):
    """Generic path at world size > 1: every rank equals an eager optimizer stepped on all_reduce-averaged
    gradients, and the replicas stay identical."""
    world, rank = hvd.size(), hvd.rank()
    torch.manual_seed(0)
    m = torch.nn.Sequential(torch.nn.Linear(6, 16), torch.nn.Tanh(), torch.nn.Linear(16, 3))
    ref = copy.deepcopy(m)

    def mk(model):
        groups = [{"params": [p for p in model.parameters() if p.dim() > 1]},
                  {"params": [p for p in model.parameters() if p.dim() == 1], "weight_decay": 0.0,
                   "adaptive": False}]
        if kind == "lars":
            return hvd.LARS(groups, lr=0.5, weight_decay=1e-3, trust_coefficient=0.01)
        return hvd.LAMB(groups, lr=0.01)

    opt = hvd.DistributedOptimizer(mk(m), named_parameters=m.named_parameters())
    assert opt.fused_engine is None
    ropt = mk(ref)
    torch.manual_seed(7)
    X, Y = torch.randn(8 * world, 6), torch.randn(8 * world, 3)
    xs, ys = X[rank * 8:(rank + 1) * 8], Y[rank * 8:(rank + 1) * 8]
    for step in range(4):
        ropt.zero_grad()
        F.mse_loss(ref(xs), ys).backward()
        for i, p in enumerate(ref.parameters()):
            p.grad.copy_(hvd.allreduce(p.grad, op=hvd.Average, name=f"ref.{step}.{i}"))
        ropt.step()
        F.mse_loss(m(xs), ys).backward()
        opt.step()
        opt.zero_grad()
    for a, b in zip(m.parameters(), ref.parameters()):
        torch.testing.assert_close(a, b, rtol=1e-5, atol=1e-7)
    return [p.detach().flatten().tolist() for p in m.parameters()]


@pytest.mark.parametrize("kind", ["lars", "lamb"])
def test_distributed_generic_path_world2(kind):
    res = run_workers(2, "test_layerwise", "gloo_trains", (kind,))
    assert res[0] == res[1], "replicas diverged"


@pytest.mark.parametrize("kind", ["lars", "lamb"])
def test_app_script_optimizer_flag_cpu(tmp_path, kind):
    env = dict(os.environ, PYTHONPATH=ROOT, B200DP_OFFLINE="1", OMP_NUM_THREADS="2")
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK"):
        env.pop(k, None)
    cmd = [sys.executable, os.path.join(ROOT, "app", "torch_train.py"), "--model", "resnet18", "--device", "cpu",
           "--epochs", "1", "--batch-size", "4", "--steps-per-epoch", "2", "--optimizer", kind]
    r = subprocess.run(cmd, cwd=str(tmp_path), env=env, capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr[-2000:]
    loss = r.stdout.split("train_loss: ")[1].split()[0]
    assert loss not in ("nan", "inf") and float(loss) == float(loss)


def test_app_script_optimizer_flag_rejects_lstm():
    sys.path.insert(0, os.path.join(ROOT, "app"))
    try:
        import torch_train
        with pytest.raises(SystemExit):
            torch_train.parse_args(["--optimizer", "lars"])
        assert torch_train.parse_args(["--model", "resnet18", "--optimizer", "lamb"]).optimizer == "lamb"
    finally:
        sys.path.remove(os.path.join(ROOT, "app"))
