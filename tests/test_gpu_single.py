"""Single-GPU tests: native library is loaded, fused update kernel (K7, world=1) vs torch
optimizers, graft smoke, app script on cuda."""
import copy
import os
import subprocess
import sys

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_native_library_loaded():
    from distributed_torch_horovod_gcp_b200.runtime import lib
    assert lib.available(), "libb200dp_comm.so missing: run __graft_entry__.build()"
    L = lib.load_comm()
    assert L is not None
    maps = open("/proc/self/maps").read()
    assert "libb200dp_comm.so" in maps


@pytest.mark.parametrize("opt_name,dtype", [("sgd", torch.float32), ("sgd", torch.bfloat16),
                                            ("adam", torch.float32), ("adamw", torch.float32)])
def test_fused_update_single_gpu(hvd_single, opt_name, dtype, monkeypatch):
    monkeypatch.setenv("B200DP_FUSED_SINGLE", "1")
    hvd = hvd_single
    dev = torch.device("cuda", 0)
    torch.manual_seed(0)
    model = torch.nn.Sequential(torch.nn.Linear(32, 100), torch.nn.ReLU(),
                                torch.nn.Linear(100, 7)).to(dev)
    ref = copy.deepcopy(model)
    model = model.to(dtype)

    def mk(ps):
        if opt_name == "sgd":
            return torch.optim.SGD(ps, lr=0.1, momentum=0.9, weight_decay=1e-2, nesterov=True)
        if opt_name == "adam":
            return torch.optim.Adam(ps, lr=1e-2)
        return torch.optim.AdamW(ps, lr=1e-2, weight_decay=0.1)
    opt = hvd.DistributedOptimizer(mk(model.parameters()), named_parameters=model.named_parameters())
    assert opt.fused_engine is not None
    ropt = mk(ref.parameters())
    x, y = torch.randn(16, 32, device=dev), torch.randn(16, 7, device=dev)
    for _ in range(5):
        if dtype == torch.float32:
            F.mse_loss(ref(x), y).backward()
        else:
            sh = copy.deepcopy(ref).to(dtype)
            F.mse_loss(sh(x.to(dtype)).float(), y).backward()
            for p, q in zip(ref.parameters(), sh.parameters()):
                p.grad = q.grad.float()
        ropt.step()
        ropt.zero_grad()
        F.mse_loss(model(x.to(dtype)).float(), y).backward()
        opt.step()
        opt.zero_grad()
    tol = dict(rtol=1e-4, atol=1e-5) if dtype == torch.float32 else dict(rtol=2e-2, atol=2e-2)
    for a, b in zip(model.parameters(), ref.parameters()):
        torch.testing.assert_close(a.float(), b, **tol)
    assert opt.fused_engine.kernel_launches == 5 * len(opt.bucket_plan())
    opt.fused_engine.export_state()
    assert len(opt.state_dict()["state"]) == 4


def test_graft_smoke():
    r = subprocess.run([sys.executable, "-c", "import __graft_entry__ as g; g.smoke()"], cwd=ROOT,
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-1500:] + r.stderr[-3000:]
    assert "smoke ok" in r.stdout


def test_app_script_cuda_single(tmp_path):
    env = dict(os.environ, PYTHONPATH=ROOT, B200DP_OFFLINE="1", B200DP_SYNTH_ROWS="2000")
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK"):
        env.pop(k, None)
    r = subprocess.run([sys.executable, os.path.join(ROOT, "app", "torch_train.py"), "--epochs", "2"],
                       cwd=str(tmp_path), env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    assert "this process is using device - cuda:0" in r.stdout
    assert r.stdout.count("train_loss") == 2 and "total training time in minutes" in r.stdout


def test_lstm_head_kernel_matches_torch():
    """K6: fused last-step gather + 3 chained linears (fp32) vs the PyTorch composition."""
    import copy
    from distributed_torch_horovod_gcp_b200.models import LSTM
    from distributed_torch_horovod_gcp_b200.ops import kernels
    dev = torch.device("cuda", 0)
    torch.manual_seed(0)
    m = LSTM(23, 10, 1, 256, device=dev)
    ref = copy.deepcopy(m)
    ref._fused = False
    x = torch.randn(32, 10, 23, device=dev)
    y = torch.randn(32, 1, 1, device=dev)
    seq = torch.empty(32, 10, 256, device=dev)
    assert kernels.enabled_for(seq) and kernels.has("lstm_fused") \
        and kernels.lstm_head_supported(seq, 9, m.linear, m.linear2, m.linear3), "fused head kernels not available"
    torch.manual_seed(1)
    out = m(x)
    torch.manual_seed(1)
    out_ref = ref(x)
    torch.testing.assert_close(out, out_ref, rtol=1e-4, atol=1e-5)
    F.mse_loss(out, y).backward()
    F.mse_loss(out_ref, y).backward()
    for (n, a), (_, b) in zip(m.named_parameters(), ref.named_parameters()):
        torch.testing.assert_close(a.grad, b.grad, rtol=2e-3, atol=1e-5, msg=lambda s: f"{n}: {s}")


def test_cuda_graph_step_matches_eager(hvd_single, monkeypatch):
    """Whole-step CUDA-graph capture (fwd + bwd + fused update kernels) == eager execution."""
    import copy
    monkeypatch.setenv("B200DP_FUSED_SINGLE", "1")
    hvd = hvd_single
    from distributed_torch_horovod_gcp_b200.utils.graph import GraphedStep
    dev = torch.device("cuda", 0)
    torch.manual_seed(0)
    base = torch.nn.Sequential(torch.nn.Linear(64, 128), torch.nn.ReLU(), torch.nn.Linear(128, 8)).to(dev)
    models = [copy.deepcopy(base) for _ in range(2)]
    opts = [hvd.DistributedOptimizer(torch.optim.SGD(m.parameters(), lr=0.05, momentum=0.9),
                                     named_parameters=m.named_parameters()) for m in models]
    assert all(o.fused_engine is not None for o in opts)

    def make_step(m, o):
        def step(x, y):
            loss = F.mse_loss(m(x), y)
            loss.backward()
            o.step()
            o.zero_grad()
            return loss.detach()
        return step

    xs = [torch.randn(16, 64, device=dev) for _ in range(6)]
    ys = [torch.randn(16, 8, device=dev) for _ in range(6)]
    eager = make_step(models[0], opts[0])
    graphed = GraphedStep(make_step(models[1], opts[1]), [xs[0], ys[0]], warmup=2)
    assert graphed.kernels_per_replay >= 1
    for _ in range(2):                       # replicate the graph's warm-up updates on the eager model
        eager(xs[0], ys[0])
    eager(xs[0], ys[0])                      # the captured step itself also executed once during capture? no:
    # capture does not execute; undo the extra eager step by re-syncing parameters instead
    with torch.no_grad():
        for a, b in zip(models[0].parameters(), models[1].parameters()):
            a.copy_(b)
    opts[0].fused_engine.params_changed()
    for ar0, ar1 in zip(opts[0].fused_engine.arenas.values(), opts[1].fused_engine.arenas.values()):
        ar0["S0"].copy_(ar1["S0"])
    opts[0].fused_engine.step_ctr.copy_(opts[1].fused_engine.step_ctr)
    for x, y in zip(xs, ys):
        le = eager(x, y)
        lg = graphed(x, y)
        torch.testing.assert_close(le, lg, rtol=1e-5, atol=1e-6)
    torch.cuda.synchronize()
    for a, b in zip(models[0].parameters(), models[1].parameters()):
        torch.testing.assert_close(a, b, rtol=1e-5, atol=1e-6)


@pytest.mark.parametrize("opt_name", ["sgd", "adam"])
def test_checkpoint_resume_fused_engine(hvd_single, monkeypatch, opt_name, tmp_path):
    """torch.save(model+optimizer state) -> fresh model/optimizer -> load -> identical continuation
    (checkpoint/resume through the fused engine's flat state arenas; SURVEY.md §5.4)."""
    import copy
    monkeypatch.setenv("B200DP_FUSED_SINGLE", "1")
    hvd = hvd_single
    dev = torch.device("cuda", 0)
    torch.manual_seed(0)

    def mk_model():
        return torch.nn.Sequential(torch.nn.Linear(32, 96), torch.nn.Tanh(), torch.nn.Linear(96, 5)).to(dev)

    def mk_opt(m):
        base = torch.optim.SGD(m.parameters(), lr=0.05, momentum=0.9, weight_decay=1e-3) \
            if opt_name == "sgd" else torch.optim.Adam(m.parameters(), lr=1e-2)
        return hvd.DistributedOptimizer(base, named_parameters=m.named_parameters())

    data = [(torch.randn(8, 32, device=dev), torch.randn(8, 5, device=dev)) for _ in range(6)]

    def run(m, o, batches):
        for x, y in batches:
            F.mse_loss(m(x), y).backward()
            o.step()
            o.zero_grad()

    m1 = mk_model()
    o1 = mk_opt(m1)
    assert o1.fused_engine is not None
    run(m1, o1, data[:3])
    ckpt = tmp_path / "ckpt.pt"
    torch.save({"model": m1.state_dict(), "opt": o1.state_dict()}, ckpt)
    sd = o1.state_dict()["state"]
    assert len(sd) == 4 and all(("momentum_buffer" in v) or ("exp_avg" in v) for v in sd.values())
    run(m1, o1, data[3:])

    m2 = mk_model()
    o2 = mk_opt(m2)
    blob = torch.load(ckpt)
    m2.load_state_dict(blob["model"])
    hvd.broadcast_parameters(m2.state_dict(), root_rank=0)      # refreshes the engine's master copy
    o2.load_state_dict(blob["opt"])
    run(m2, o2, data[3:])
    for a, b in zip(m1.parameters(), m2.parameters()):
        torch.testing.assert_close(a, b, rtol=1e-5, atol=1e-6)
