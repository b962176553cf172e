"""Worker bodies for the sequence-parallel group tests (``mp_util.run_workers``): every rank runs one of these with
``hvd`` initialised.  Groups are the contiguous blocks of G ranks; group k draws its tokens with seed 1 + k.  CPU
cases run over Gloo on the reference path; ``kernel_*`` cases need one GPU per rank."""
import torch

from distributed_torch_horovod_gcp_b200.models import gpt_tiny
from distributed_torch_horovod_gcp_b200.ops import seq_parallel as sp
from sp_cases import _tokens


def _group_batches(B, S, vocab, groups):
    """Every group's (inputs, targets), group k from seed 1 + k."""
    return [_tokens(B, S, vocab, seed=1 + k) for k in range(groups)]


def _grad_err(model, full):
    err = 0.0
    for (n, p), q in zip(model.named_parameters(), full.parameters()):
        assert p.grad is not None, n
        err = max(err, float((p.grad - q.grad).abs().max() / q.grad.abs().max().clamp_min(1e-12)))
    return err


def gpt_groups_match_full(hvd, B, S, G):
    """gpt_tiny(sequence_parallel=True, sequence_parallel_size=G) on this rank's shard of its group's batch against
    one full-sequence model run on the batches of all groups together: each group's mean loss against the full
    model's loss on that group's batch, the world's mean loss against its loss on all batches, and the gradients
    after DistributedOptimizer's averaging over the world against its gradients on all batches."""
    rank, world = hvd.rank(), hvd.size()
    k, gr = rank // G, rank % G
    torch.manual_seed(0)
    full = gpt_tiny()
    model = gpt_tiny(sequence_parallel=True, sequence_parallel_size=G)
    model.load_state_dict(full.state_dict())
    batches = _group_batches(B, S, full.vocab, world // G)
    with torch.no_grad():
        group_full = [float(full(i, t)) for i, t in batches]
    full_loss = full(torch.cat([i for i, _ in batches]), torch.cat([t for _, t in batches]))
    full_loss.backward()
    opt = hvd.DistributedOptimizer(torch.optim.SGD(model.parameters(), lr=0.0),
                                   named_parameters=model.named_parameters())
    idx, tgt = batches[k]
    shard = (lambda t: sp.zigzag_shard(t, 1, gr, G))
    loss = model(shard(idx), shard(tgt))
    loss.backward()
    opt.synchronize()
    losses = hvd.allgather(loss.detach().view(1))
    group_mean = float(losses[k * G:(k + 1) * G].mean())
    return {"loss": float(full_loss), "group_loss": group_full[k],
            "group_loss_err": abs(group_mean - group_full[k]),
            "loss_err": abs(float(losses.mean()) - float(full_loss)),
            "grad_rel_err": _grad_err(model, full)}


def gpt_whole_world_size_is_default(hvd, B, S):
    """sequence_parallel_size=world against sequence_parallel_size=None: the same loss and gradients, bit for bit."""
    rank, world = hvd.rank(), hvd.size()
    torch.manual_seed(0)
    a = gpt_tiny(sequence_parallel=True)
    b = gpt_tiny(sequence_parallel=True, sequence_parallel_size=world)
    b.load_state_dict(a.state_dict())
    idx, tgt = _tokens(B, S, a.vocab)
    shard = (lambda t: sp.zigzag_shard(t, 1, rank, world))
    out = []
    for m in (a, b):
        loss = m(shard(idx), shard(tgt))
        loss.backward()
        out.append((loss.detach(), [p.grad for p in m.parameters()]))
    same = torch.equal(out[0][0], out[1][0]) and all(torch.equal(x, y) for x, y in zip(out[0][1], out[1][1]))
    return same


def refusals(hvd):
    """The ValueErrors of GPT(sequence_parallel_size=...) and sp_attention over a group, by name."""
    world = hvd.size()
    out = []
    for name, kw in (("not a divisor", dict(sequence_parallel=True, sequence_parallel_size=world - 1)),
                     ("zero", dict(sequence_parallel=True, sequence_parallel_size=0)),
                     ("negative", dict(sequence_parallel=True, sequence_parallel_size=-2)),
                     ("without sequence_parallel", dict(sequence_parallel_size=2)),
                     ("dropout", dict(sequence_parallel=True, sequence_parallel_size=2, dropout=0.1))):
        try:
            gpt_tiny(**kw)
        except ValueError:
            out.append(name)
    ps = gpt_tiny(sequence_parallel=True, sequence_parallel_size=2)._sp_set
    q = torch.randn(1, 2, 8, 64)
    try:
        sp.sp_attention(q, q, q, True, 0.1, process_set=ps)
    except ValueError:
        out.append("attention dropout")
    return out


def group_sets_reused(hvd, G):
    """Two models with sequence_parallel_size=G: the second registers no new process set and holds the first's."""
    from distributed_torch_horovod_gcp_b200 import _state
    sets = _state.runtime().process_sets
    first = gpt_tiny(sequence_parallel=True, sequence_parallel_size=G)
    n = len(sets)
    second = gpt_tiny(sequence_parallel=True, sequence_parallel_size=G)
    return {"added": n, "again": len(sets) - n, "same": second._sp_set is first._sp_set,
            "ranks": first._sp_set.ranks}


# ------------------------------------------------------------------ one GPU per rank
def kernel_gpt_groups_match_reference(hvd, B, S, G):
    """A bf16 gpt_tiny with sequence_parallel_size=G on the kernel path (S / G a multiple of 256) against an fp32
    copy of it, whose attention takes the reference path (all-gather over the group's torch.distributed group and
    SDPA with a mask): the loss and the gradients within the bf16 tolerances of ``sp_cases.kernel_gpt_step``."""
    from distributed_torch_horovod_gcp_b200.ops import counters
    rank, world = hvd.rank(), hvd.size()
    k, gr = rank // G, rank % G
    dev = torch.device("cuda", torch.cuda.current_device())
    torch.manual_seed(0)
    model = gpt_tiny(context=S, sequence_parallel=True, sequence_parallel_size=G).to(dev).to(torch.bfloat16)
    ref = gpt_tiny(context=S, sequence_parallel=True, sequence_parallel_size=G).to(dev)
    ref.load_state_dict({n: t.float() for n, t in model.state_dict().items()})
    idx, tgt = [t.to(dev) for t in _group_batches(B, S, model.vocab, world // G)[k]]
    shard = (lambda t: sp.zigzag_shard(t, 1, gr, G))
    n0 = counters.snapshot().get("attn_sp_fwd", 0)
    loss = model(shard(idx), shard(tgt))
    loss.backward()
    torch.cuda.synchronize()
    assert counters.snapshot().get("attn_sp_fwd", 0) > n0, "the bf16 model did not take the kernel path"
    ref_loss = ref(shard(idx), shard(tgt))
    ref_loss.backward()
    # each rank's loss is the mean over its own shard; a group's mean over its ranks is the loss of its batch
    refs = hvd.allgather(ref_loss.detach().float().view(1))
    lerr = abs(float(loss) - float(ref_loss))
    assert lerr <= 2e-2 * abs(float(ref_loss)), (float(loss), float(ref_loss))
    num = sum(float((p.grad.double() - q.grad.double()).norm() ** 2) for p, q in zip(model.parameters(),
                                                                                     ref.parameters()))
    den = sum(float(q.grad.double().norm() ** 2) for q in ref.parameters())
    rel = (num / max(den, 1e-30)) ** 0.5
    assert rel < 5e-2, rel
    return {"group": k, "loss": float(loss), "ref": float(ref_loss), "grad_rel_err": rel,
            "group_ref": float(refs[k * G:(k + 1) * G].mean())}
