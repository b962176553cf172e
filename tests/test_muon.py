"""``hvd.Muon`` without a GPU: Muon groups against ``torch.optim.Muon`` and AdamW groups against
``torch.optim.AdamW``, bit for bit; argument validation; the generic DistributedOptimizer path over Gloo; and the
training script's ``--optimizer muon``."""
import copy
import os
import subprocess
import sys

import pytest
import torch
import torch.nn.functional as F

from mp_util import run_workers

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SHAPES = [(24, 16), (16, 40), (32, 32)]      # tall, wide, square


def _params(seed=0):
    torch.manual_seed(seed)
    return [torch.nn.Parameter(torch.randn(*s)) for s in SHAPES]


def _run(opt, ps, steps=4, seed=1):
    g = torch.Generator().manual_seed(seed)
    for _ in range(steps):
        for p in ps:
            p.grad = torch.randn(p.shape, generator=g)
        opt.step()


@pytest.mark.parametrize("nesterov", [True, False])
@pytest.mark.parametrize("adjust_lr_fn", [None, "original", "match_rms_adamw"])
def test_muon_groups_match_torch_muon(nesterov, adjust_lr_fn):
    import distributed_torch_horovod_gcp_b200.torch as hvd
    kw = dict(lr=0.02, weight_decay=0.1, momentum=0.9, nesterov=nesterov, adjust_lr_fn=adjust_lr_fn)
    a, b = _params(), _params()
    opt, ref = hvd.Muon(a, **kw), torch.optim.Muon(b, **kw)
    _run(opt, a)
    _run(ref, b)
    for x, y in zip(a, b):
        assert torch.equal(x, y)
        assert torch.equal(opt.state[x]["momentum_buffer"], ref.state[y]["momentum_buffer"])


def test_muon_state_and_ns_settings_match_torch():
    import distributed_torch_horovod_gcp_b200.torch as hvd
    kw = dict(lr=0.01, weight_decay=0.0, ns_steps=3, ns_coefficients=(3.0, -3.2, 1.2), eps=1e-5)
    a, b = _params(3), _params(3)
    opt, ref = hvd.Muon(a, **kw), torch.optim.Muon(b, **kw)
    _run(opt, a, steps=3)
    _run(ref, b, steps=3)
    for x, y in zip(a, b):
        assert torch.equal(x, y)
        assert torch.equal(opt.state[x]["momentum_buffer"], ref.state[y]["momentum_buffer"])


def test_adamw_groups_match_torch_adamw():
    import distributed_torch_horovod_gcp_b200.torch as hvd
    torch.manual_seed(0)
    shapes = [(7, 5), (13,), (3, 4, 2)]
    a = [torch.nn.Parameter(torch.randn(*s)) for s in shapes]
    b = [torch.nn.Parameter(p.detach().clone()) for p in a]
    opt = hvd.Muon([{"params": a, "use_muon": False}], lr=3e-3, weight_decay=0.05, betas=(0.8, 0.97), adam_eps=1e-6)
    ref = torch.optim.AdamW(b, lr=3e-3, weight_decay=0.05, betas=(0.8, 0.97), eps=1e-6)
    _run(opt, a, steps=5)
    _run(ref, b, steps=5)
    for x, y in zip(a, b):
        assert torch.equal(x, y)
        for key in ("step", "exp_avg", "exp_avg_sq"):
            assert torch.equal(opt.state[x][key], ref.state[y][key]), key


def test_mixed_groups_follow_their_own_rules():
    import distributed_torch_horovod_gcp_b200.torch as hvd
    torch.manual_seed(0)
    m = [torch.nn.Parameter(torch.randn(16, 24)), torch.nn.Parameter(torch.randn(8))]
    mm, ma = [torch.nn.Parameter(m[0].detach().clone())], [torch.nn.Parameter(m[1].detach().clone())]
    opt = hvd.Muon([{"params": [m[0]]}, {"params": [m[1]], "use_muon": False, "weight_decay": 0.0}], lr=0.01)
    _run(opt, m, steps=3)
    g = torch.Generator().manual_seed(1)
    r1, r2 = torch.optim.Muon(mm, lr=0.01), torch.optim.AdamW(ma, lr=0.01, weight_decay=0.0, betas=(0.9, 0.95),
                                                             eps=1e-8)
    for _ in range(3):
        mm[0].grad = torch.randn(mm[0].shape, generator=g)
        ma[0].grad = torch.randn(ma[0].shape, generator=g)
        r1.step()
        r2.step()
    assert torch.equal(m[0], mm[0]) and torch.equal(m[1], ma[0])


@pytest.mark.parametrize("kwargs", [{"lr": -1.0}, {"weight_decay": -0.1}, {"eps": -1e-7}, {"adam_eps": -1e-8},
                                    {"momentum": -0.1}, {"momentum": 1.0}, {"ns_steps": 0}, {"ns_steps": 100},
                                    {"adjust_lr_fn": "rms"}, {"betas": (1.0, 0.9)}, {"betas": (0.9, -0.1)},
                                    {"maximize": True}])
def test_rejects_bad_arguments(kwargs):
    import distributed_torch_horovod_gcp_b200.torch as hvd
    with pytest.raises(ValueError):
        hvd.Muon([torch.nn.Parameter(torch.randn(4, 4))], **kwargs)


def test_rejects_non_matrix_in_muon_group_and_bad_added_group():
    import distributed_torch_horovod_gcp_b200.torch as hvd
    lin = torch.nn.Linear(4, 4)
    with pytest.raises(ValueError):
        hvd.Muon(lin.parameters())
    with pytest.raises(ValueError):
        hvd.Muon([{"params": [torch.nn.Parameter(torch.randn(2, 2, 2))]}])
    opt = hvd.Muon([{"params": [lin.weight]}, {"params": [lin.bias], "use_muon": False}])
    with pytest.raises(ValueError):
        opt.add_param_group({"params": [torch.nn.Parameter(torch.randn(3, 3))], "ns_steps": 0})
    with pytest.raises(ValueError):
        opt.add_param_group({"params": [torch.nn.Parameter(torch.randn(3))]})


def test_classified_for_the_fused_engine():
    import distributed_torch_horovod_gcp_b200.torch as hvd
    from distributed_torch_horovod_gcp_b200.parallel.fused_engine import _classify
    assert _classify(hvd.Muon([torch.nn.Parameter(torch.randn(8, 8))])) == "muon"
    assert _classify(torch.optim.Muon([torch.nn.Parameter(torch.randn(8, 8))])) is None


def gloo_trains(hvd):
    """Generic path at world size 2: every rank equals an eager hvd.Muon stepped on all_reduce-averaged
    gradients, and the replicas stay identical."""
    world, rank = hvd.size(), hvd.rank()
    torch.manual_seed(0)
    m = torch.nn.Sequential(torch.nn.Linear(8, 16), torch.nn.Tanh(), torch.nn.Linear(16, 4))
    ref = copy.deepcopy(m)

    def mk(model):
        return hvd.Muon([{"params": [p for p in model.parameters() if p.dim() == 2]},
                         {"params": [p for p in model.parameters() if p.dim() < 2], "use_muon": False,
                          "weight_decay": 0.0}], lr=0.02)

    opt = hvd.DistributedOptimizer(mk(m), named_parameters=m.named_parameters())
    assert opt.fused_engine is None
    ropt = mk(ref)
    torch.manual_seed(7)
    X, Y = torch.randn(8 * world, 8), torch.randn(8 * world, 4)
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
        torch.testing.assert_close(a, b, rtol=1e-5, atol=1e-6)
    return [p.detach().flatten().tolist() for p in m.parameters()]


def test_distributed_generic_path_world2():
    res = run_workers(2, "test_muon", "gloo_trains", ())
    assert res[0] == res[1], "replicas diverged"


def test_app_script_muon_trains_gpt_tiny(tmp_path):
    env = dict(os.environ, PYTHONPATH=ROOT, B200DP_OFFLINE="1", OMP_NUM_THREADS="2")
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK"):
        env.pop(k, None)
    cmd = [sys.executable, os.path.join(ROOT, "app", "torch_train.py"), "--model", "gpt-tiny", "--device", "cpu",
           "--epochs", "1", "--batch-size", "2", "--steps-per-epoch", "2", "--optimizer", "muon"]
    r = subprocess.run(cmd, cwd=str(tmp_path), env=env, capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr[-2000:]
    loss = r.stdout.split("train_loss: ")[1].split()[0]
    assert loss not in ("nan", "inf") and float(loss) == float(loss)


def test_app_script_muon_groups_and_refusal():
    sys.path.insert(0, os.path.join(ROOT, "app"))
    try:
        import torch_train
        from distributed_torch_horovod_gcp_b200.models import build
        for model in ("resnet18", "lstm", "vit-tiny"):
            with pytest.raises(SystemExit):
                torch_train.parse_args(["--model", model, "--optimizer", "muon"])
        assert torch_train.parse_args(["--model", "gpt-tiny", "--optimizer", "muon"]).optimizer == "muon"
        m = build("gpt-tiny")
        opt = torch_train.gpt_muon_optimizer(m, 1e-3)
        names = {id(p): n for n, p in m.named_parameters()}
        muon = [names[id(p)] for g in opt.param_groups if g["use_muon"] for p in g["params"]]
        assert len(muon) == 4 * len(m.layers)
        assert all(n.split(".")[-2] in ("qkv", "proj", "fc1", "fc2") for n in muon)
        assert all(g["adjust_lr_fn"] == "match_rms_adamw" for g in opt.param_groups)
        assert sum(len(g["params"]) for g in opt.param_groups) == len(names)
    finally:
        sys.path.remove(os.path.join(ROOT, "app"))


@pytest.mark.parametrize("missing", ["gemm", "gemm_scaled"])
def test_fused_engine_needs_the_scaled_gemm_entry_point(monkeypatch, missing):
    """A kernels library without the GEMM or without its scaled-residual entry point sends Muon to the generic
    path (with a reason to log) instead of failing inside a backward hook."""
    import distributed_torch_horovod_gcp_b200.torch as hvd
    from distributed_torch_horovod_gcp_b200.ops import kernels
    from distributed_torch_horovod_gcp_b200.parallel.fused_engine import _muon_unsupported
    monkeypatch.setattr(kernels, "has", lambda op: op != missing)
    opt = hvd.Muon([torch.nn.Parameter(torch.randn(8, 16))])
    assert "scaled-residual" in _muon_unsupported(opt, [])
    monkeypatch.setattr(kernels, "has", lambda op: True)
    assert _muon_unsupported(opt, []) is None
