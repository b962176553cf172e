"""Worker bodies for the gradient-clipping tests (``max_grad_norm=``): the generic path over Gloo (CPU) and
the fused engine on several GPUs.  Each function runs on every rank."""
import copy
import hashlib

import torch
import torch.distributed as dist
import torch.nn.functional as F


def _model(seed):
    torch.manual_seed(seed)
    return torch.nn.Sequential(torch.nn.Linear(6, 16), torch.nn.Tanh(), torch.nn.Linear(16, 3))


def _mk(opt_name, params):
    if opt_name == "sgd":
        return torch.optim.SGD(params, lr=0.1, momentum=0.9, weight_decay=1e-3, nesterov=True)
    if opt_name == "adam":
        return torch.optim.Adam(params, lr=1e-2)
    return torch.optim.AdamW(params, lr=1e-2, weight_decay=0.1)


def generic_matches_torch(hvd, opt_name, max_norm):
    """Generic path (and, at size 1, the plain optimizer): parameters and ``grad_norm`` equal
    ``clip_grad_norm_`` on the all_reduce-averaged gradients followed by the torch optimizer."""
    world, rank = hvd.size(), hvd.rank()
    torch.manual_seed(7)
    X, Y = torch.randn(8 * world, 6), torch.randn(8 * world, 3)
    m = _model(0)
    ref = copy.deepcopy(m)
    opt = hvd.DistributedOptimizer(_mk(opt_name, m.parameters()), named_parameters=m.named_parameters(),
                                   max_grad_norm=max_norm)
    ropt = _mk(opt_name, ref.parameters())
    hvd.broadcast_parameters(m.state_dict(), root_rank=0)
    assert opt.grad_norm is not None and opt.grad_norm.dtype == torch.float32 and opt.grad_norm.dim() == 0
    norm_ptr = opt.grad_norm.data_ptr()
    norms = []
    for step in range(3):
        xs, ys = X[rank * 8:(rank + 1) * 8], Y[rank * 8:(rank + 1) * 8]
        ropt.zero_grad()
        F.mse_loss(ref(xs), ys).backward()
        for i, p in enumerate(ref.parameters()):
            p.grad.copy_(hvd.allreduce(p.grad, op=hvd.Average, name=f"ref.{step}.{i}"))
        rn = torch.nn.utils.clip_grad_norm_(ref.parameters(), max_norm)
        ropt.step()
        F.mse_loss(m(xs), ys).backward()
        opt.step()
        opt.zero_grad()
        assert float(rn) > max_norm, "the test must clip on every step"
        torch.testing.assert_close(opt.grad_norm, rn.float(), rtol=1e-6, atol=0.0)
        assert opt.grad_norm.data_ptr() == norm_ptr
        norms.append(float(opt.grad_norm))
    for a, b in zip(m.parameters(), ref.parameters()):
        torch.testing.assert_close(a, b, rtol=1e-5, atol=1e-7)
    return norms


def unset_and_invalid(hvd):
    m = _model(0)
    opt = hvd.DistributedOptimizer(torch.optim.SGD(m.parameters(), lr=0.1), named_parameters=m.named_parameters())
    assert opt.grad_norm is None
    m(torch.randn(4, 6)).sum().backward()
    opt.step()
    assert opt.grad_norm is None
    for bad in (0, 0.0, -1, -1.0, float("inf"), float("-inf"), float("nan"), "1.0", True):
        try:
            hvd.DistributedOptimizer(torch.optim.SGD(m.parameters(), lr=0.1),
                                     named_parameters=m.named_parameters(), max_grad_norm=bad)
        except ValueError:
            continue
        raise AssertionError(f"max_grad_norm={bad!r} was accepted")
    return True


# ------------------------------------------------------------------ multi-GPU (fused engine, symmetric runtime)
def fused_clip_matches_nccl(hvd, opt_name):
    """The method of bench.py's selfcheck, in clip mode: IDENTICAL local gradients on both arms; (a) NCCL
    all_reduce average + clip_grad_norm_ + the torch optimizer on a plain clone, (b) the same gradients in
    the fused engine's buckets, one step.  Returns the norm and a digest of the updated parameters, which
    the caller compares across ranks."""
    from distributed_torch_horovod_gcp_b200 import _state
    assert _state.get_symm() is not None, f"symmetric runtime unavailable: {_state.runtime().symm_failed}"
    r, n = hvd.rank(), hvd.size()
    dev = torch.device("cuda", torch.cuda.current_device())
    torch.manual_seed(0)
    model = torch.nn.Sequential(torch.nn.Linear(64, 300), torch.nn.Tanh(), torch.nn.Linear(300, 257),
                                torch.nn.Tanh(), torch.nn.Linear(257, 8)).to(dev)
    max_norm = 0.05
    opt = hvd.DistributedOptimizer(_mk(opt_name, model.parameters()), named_parameters=model.named_parameters(),
                                   bucket_bytes=128 << 10, max_grad_norm=max_norm)
    assert opt.fused_engine is not None and opt.fused_engine.clip
    assert set(opt.fused_engine.algorithms().values()) == {"oneshot"}
    hvd.broadcast_parameters(model.state_dict(), root_rank=0)
    ref = copy.deepcopy(model)
    for p in ref.parameters():
        p.grad = None
        if hasattr(p, "_b200dp_sink"):
            del p._b200dp_sink
    ropt = _mk(opt_name, ref.parameters())
    norms = []
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
        rn = torch.nn.utils.clip_grad_norm_(ref.parameters(), max_norm)
        ropt.step()
        torch.cuda.synchronize()
        assert float(rn) > max_norm
        torch.testing.assert_close(opt.grad_norm, rn, rtol=1e-5, atol=0.0)
        norms.append(opt.grad_norm.item())
    for a, b in zip(model.parameters(), ref.parameters()):
        torch.testing.assert_close(a, b, rtol=2e-4, atol=2e-5)
    h = hashlib.sha256()
    for p in model.parameters():
        h.update(p.detach().contiguous().view(torch.uint8).cpu().numpy().tobytes())
    got = [None] * n
    dist.all_gather_object(got, (norms, h.hexdigest()))
    assert all(g[0] == got[0][0] for g in got), f"grad_norm differs across ranks: {got}"
    assert all(g[1] == got[0][1] for g in got), "replicas diverged"
    opt.remove_hooks()
    return norms, h.hexdigest()
