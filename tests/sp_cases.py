"""Worker bodies for the sequence-parallel tests (``mp_util.run_workers``): every rank runs one of these with
``hvd`` initialised.  CPU cases run over Gloo on the reference path; ``kernel_*`` cases need one GPU per rank."""
import copy

import torch

from distributed_torch_horovod_gcp_b200.models import gpt_tiny
from distributed_torch_horovod_gcp_b200.ops import seq_parallel as sp


def _tokens(B, S, vocab, seed=1):
    t = torch.randint(0, vocab, (B, S + 1), generator=torch.Generator().manual_seed(seed))
    return t[:, :-1], t[:, 1:]


def _rel(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm().clamp_min(1e-30))


def gpt_matches_full(hvd, B, S):
    """gpt_tiny(sequence_parallel=True) on this rank's shard against the full-sequence model run on every rank:
    the loss averaged over ranks and the gradients after DistributedOptimizer's averaging.  Returns the loss error
    and the largest gradient error relative to each tensor's largest gradient."""
    rank, world = hvd.rank(), hvd.size()
    torch.manual_seed(0)
    full = gpt_tiny()
    model = gpt_tiny(sequence_parallel=True)
    model.load_state_dict(full.state_dict())
    idx, tgt = _tokens(B, S, full.vocab)
    full_loss = full(idx, tgt)
    full_loss.backward()
    opt = hvd.DistributedOptimizer(torch.optim.SGD(model.parameters(), lr=0.0),
                                   named_parameters=model.named_parameters())
    shard = (lambda t: sp.zigzag_shard(t, 1, rank, world))
    loss = model(shard(idx), shard(tgt))
    loss.backward()
    opt.synchronize()
    avg = hvd.allreduce(loss.detach(), average=True)
    loss_err = abs(float(avg) - float(full_loss))
    grad_err = 0.0
    for (n, p), q in zip(model.named_parameters(), full.parameters()):
        assert p.grad is not None, n
        grad_err = max(grad_err, float((p.grad - q.grad).abs().max() / q.grad.abs().max().clamp_min(1e-12)))
    return {"loss": float(full_loss), "loss_err": loss_err, "grad_rel_err": grad_err}


def dropout_refused(hvd):
    """sp_attention with dropout_p > 0 and GPT(sequence_parallel=True, dropout > 0) raise ValueError."""
    q = torch.randn(1, 2, 8, 64)
    out = []
    try:
        sp.sp_attention(q, q, q, True, 0.1)
    except ValueError:
        out.append("op")
    try:
        gpt_tiny(sequence_parallel=True, dropout=0.1)
    except ValueError:
        out.append("model")
    return out


# ------------------------------------------------------------------ one GPU per rank
def kernel_attention_matches_full(hvd, B, H, S, causal):
    """The kernel path of sp_attention on this rank's shard against attention_fused on the full sequence run on
    this GPU: O, dK and dV bit for bit, dQ within the float64 bounds of the full-sequence kernel."""
    from distributed_torch_horovod_gcp_b200.ops import attention, counters
    from fp64_bounds import assert_within_bound
    from test_gpu_causal_attention import causal_bwd_bounds
    from test_gpu_vit_numerics import attn_bwd_bounds
    rank, world = hvd.rank(), hvd.size()
    g = torch.Generator().manual_seed(5)
    q, k, v, do = [torch.randn(B, H, S, 64, generator=g).bfloat16().cuda() for _ in range(4)]
    leaves = [t.clone().requires_grad_(True) for t in (q, k, v)]
    o_full = attention.attention_fused(*leaves, causal=causal)
    o_full.backward(do)
    shard = (lambda t: sp.zigzag_shard(t, 2, rank, world))
    mine = [shard(t).requires_grad_(True) for t in (q, k, v)]
    n0 = counters.snapshot().get("attn_sp_fwd", 0)
    o = sp.sp_attention(*mine, causal=causal)
    o.backward(shard(do))
    torch.cuda.synchronize()
    assert counters.snapshot().get("attn_sp_fwd", 0) == n0 + 1, "sp_attention did not take the kernel path"
    assert torch.equal(o.detach(), shard(o_full.detach())), "O differs from the full-sequence kernel's rows"
    for name, got, ref in (("dk", mine[1].grad, leaves[1].grad), ("dv", mine[2].grad, leaves[2].grad)):
        assert torch.equal(got, shard(ref)), f"{name} differs from the full-sequence kernel's rows"
    bounds = (causal_bwd_bounds if causal else attn_bwd_bounds)(q, k, v, do, o_full.detach())
    dq_ref, dq_b = bounds[0]
    assert_within_bound(mine[0].grad, shard(dq_ref), group="sp dq (multi-GPU)", terms=[(1.0, shard(dq_b))])
    return True


def kernel_gpt_step(hvd, B, S):
    """One fused-engine SGD step of a bf16 GPT with sequence parallelism against one plain SGD step of the
    full-sequence model on this GPU: the rank-averaged loss and the parameter updates close to the full-sequence
    ones, and parameters bit-identical across ranks after the update."""
    rank, world = hvd.rank(), hvd.size()
    dev = torch.device("cuda", torch.cuda.current_device())
    torch.manual_seed(0)
    full = gpt_tiny(context=S).to(dev).to(torch.bfloat16)
    model = copy.deepcopy(full)
    model.sequence_parallel = True
    start = [p.detach().clone() for p in full.parameters()]
    lr = 1.0
    idx, tgt = [t.to(dev) for t in _tokens(B, S, full.vocab)]
    full_loss = full(idx, tgt)
    full_loss.backward()
    torch.optim.SGD(full.parameters(), lr=lr).step()
    opt = hvd.DistributedOptimizer(torch.optim.SGD(model.parameters(), lr=lr),
                                   named_parameters=model.named_parameters())
    shard = (lambda t: sp.zigzag_shard(t, 1, rank, world))
    loss = model(shard(idx), shard(tgt))
    loss.backward()
    opt.step()
    torch.cuda.synchronize()
    assert opt.fused_engine is not None, "the fused engine did not run"
    avg = float(hvd.allreduce(loss.detach().float(), average=True))
    assert abs(avg - float(full_loss)) <= 2e-2 * abs(float(full_loss)), (avg, float(full_loss))
    step_sp = torch.cat([(p.detach().double() - s0.double()).reshape(-1) for p, s0 in zip(model.parameters(), start)])
    step_full = torch.cat([(f.detach().double() - s0.double()).reshape(-1) for f, s0 in zip(full.parameters(), start)])
    worst = _rel(step_sp, step_full)
    assert worst < 5e-2, worst
    flat = torch.cat([p.detach().float().reshape(-1) for p in model.parameters()])
    gathered = hvd.allgather(flat.view(1, -1))
    assert all(torch.equal(gathered[0], gathered[r]) for r in range(world)), "replicas diverged"
    return {"loss": avg, "full": float(full_loss), "update_rel_err": worst}
