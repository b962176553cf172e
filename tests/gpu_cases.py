"""Worker bodies for the multi-GPU tests (one process per GPU, symmetric-memory kernels)."""
import copy
import os

import torch
import torch.distributed as dist
import torch.nn.functional as F


def _symm(hvd):
    from distributed_torch_horovod_gcp_b200 import _state
    s = _state.get_symm()
    assert s is not None, f"symmetric runtime unavailable: {_state.runtime().symm_failed}"
    return s


def runtime_setup(hvd):
    """cuMem allocation + fd exchange + peer mapping (+ multicast) works; peers see writes."""
    s = _symm(hvd)
    r, n = hvd.rank(), hvd.size()
    buf = s.alloc(1 << 20)
    t = buf.tensor(torch.float32)
    t.fill_(float(r + 1))
    torch.cuda.synchronize()
    hvd.barrier()
    # read every peer's buffer through the peer mapping
    from distributed_torch_horovod_gcp_b200.runtime.symm import _Raw
    for q in range(n):
        peer = torch.as_tensor(_Raw(buf.peer_ptrs[q], 1024, buf), device=s.device).view(torch.float32)
        assert float(peer[0]) == q + 1 and float(peer[-1]) == q + 1, (q, peer[:4])
    hvd.barrier()
    return {"multicast": bool(s.multicast), "mc_ptr": buf.mc_ptr != 0, "gran": s.gran,
            "mc_gran": s.mc_gran, "sms": s.sm_count, "cc": s.cc}


def allreduce_matches_nccl(hvd, algos):
    s = _symm(hvd)
    from distributed_torch_horovod_gcp_b200.runtime import symm as S
    r, n = hvd.rank(), hvd.size()
    dev = s.device
    results = {}
    sizes = [1, 3, 4, 64, 1000, 4096 + 1, 65536, 370049, 1 << 20, (4 << 20) + 12]
    for dtype, tol in ((torch.float32, 1e-5), (torch.bfloat16, 2e-2), (torch.float16, 2e-3)):
        for numel in sizes:
            torch.manual_seed(numel * 7 + r)
            x = torch.randn(numel, device=dev).to(dtype)
            ref = x.clone().float()
            dist.all_reduce(ref)                 # NCCL oracle in fp32
            ref = ref / n
            for algo in algos:
                if algo == "nvls" and not s.multicast:
                    continue
                code = {"oneshot": S.ALGO_ONESHOT, "twoshot": S.ALGO_TWOSHOT, "nvls": S.ALGO_NVLS}[algo]
                y = x.clone()
                ev = s.allreduce_(y, postscale=1.0 / n, algo=code)
                ev.synchronize()
                err = (y.float() - ref).abs().max().item() / max(ref.abs().max().item(), 1e-6)
                assert err < tol, (dtype, numel, algo, err)
                # replicas bit-identical across ranks
                g = [torch.empty_like(y) for _ in range(n)]
                dist.all_gather(g, y)
                assert all(torch.equal(g[0], q) for q in g), (dtype, numel, algo)
                results[(str(dtype), numel, algo)] = err
    # public API, default algo choice, Sum / Average / prescale, non-contiguous, symmetric tensor
    t = torch.full((5, 7), float(r + 1), device=dev)
    out = hvd.allreduce(t, op=hvd.Sum)
    assert torch.all(out == sum(range(1, n + 1)))
    out = hvd.allreduce(t.t(), prescale_factor=2.0)
    assert torch.allclose(out, torch.full((7, 5), 2.0 * sum(range(1, n + 1)) / n, device=dev))
    st = hvd.symm_empty(1 << 16, torch.float32)
    st.fill_(float(r))
    hvd.allreduce_(st, op=hvd.Sum)
    torch.cuda.synchronize()
    assert torch.all(st == sum(range(n)))
    s.check_errors()
    return len(results)


def broadcast_matches(hvd):
    s = _symm(hvd)
    r, n = hvd.rank(), hvd.size()
    dev = s.device
    for numel in (1, 5, 1024, 370049, (2 << 20) + 3):
        for root in sorted({0, n - 1}):
            x = torch.arange(numel, device=dev, dtype=torch.float32) + 1000.0 * r
            hvd.broadcast_(x, root)
            torch.cuda.synchronize()
            want = torch.arange(numel, device=dev, dtype=torch.float32) + 1000.0 * root
            assert torch.equal(x, want), (numel, root)
    from distributed_torch_horovod_gcp_b200.models import LSTM, resnet18
    m = LSTM(23, 10, 1, 256, device=dev)
    with torch.no_grad():
        for p in m.parameters():
            p.add_(float(r))
    hvd.broadcast_parameters(m.state_dict(), root_rank=0)
    m2 = resnet18(num_classes=10, small_input=True).to(dev)
    m2.bn1.running_mean.fill_(float(r))
    hvd.broadcast_parameters(m2.state_dict(), root_rank=0)       # params + BN buffers (int64 too)
    flat = torch.cat([v.reshape(-1).float() for v in list(m.state_dict().values()) +
                      list(m2.state_dict().values())])
    g = [torch.empty_like(flat) for _ in range(n)]
    dist.all_gather(g, flat)
    assert all(torch.equal(g[0], q) for q in g)
    assert float(m2.bn1.running_mean[0]) == 0.0
    s.check_errors()
    return True


def fused_optimizer_matches_torch(hvd, opt_name, dtype_name, algo):
    """N-rank fused allreduce+update == single-process torch optimizer on the averaged grads."""
    os.environ["B200DP_ALGO"] = algo
    s = _symm(hvd)
    s.algo_override = algo
    r, n = hvd.rank(), hvd.size()
    dev = s.device
    dtype = {"fp32": torch.float32, "bf16": torch.bfloat16}[dtype_name]
    torch.manual_seed(0)
    model = torch.nn.Sequential(torch.nn.Linear(64, 300), torch.nn.Tanh(),
                                torch.nn.Linear(300, 257), torch.nn.Tanh(),
                                torch.nn.Linear(257, 8)).to(dev)
    ref = copy.deepcopy(model).float()
    model = model.to(dtype)

    def mk(params):
        if opt_name == "sgd":
            return torch.optim.SGD(params, lr=0.05, momentum=0.9, weight_decay=1e-3)
        if opt_name == "sgd_nesterov":
            return torch.optim.SGD(params, lr=0.05, momentum=0.8, nesterov=True)
        if opt_name == "adam":
            return torch.optim.Adam(params, lr=1e-2, weight_decay=1e-2)
        return torch.optim.AdamW(params, lr=1e-2, weight_decay=1e-2)
    opt = hvd.DistributedOptimizer(mk(model.parameters()), named_parameters=model.named_parameters(),
                                   bucket_bytes=256 << 10)
    assert opt.fused_engine is not None, "fused engine not created"
    assert isinstance(opt, type(mk(ref.parameters())))
    ropt = mk(ref.parameters())
    hvd.broadcast_parameters(model.state_dict(), root_rank=0)
    torch.manual_seed(5)
    X = torch.randn(4 * n, 64, device=dev)
    Y = torch.randn(4 * n, 8, device=dev)
    for step in range(4):
        # reference: fp32 model, grads computed from the SAME low-precision forward as the DP ranks
        ropt.zero_grad()
        if dtype == torch.float32:
            F.mse_loss(ref(X), Y).backward()
        else:
            # emulate: each rank's bf16 grads, averaged in fp32
            shadow = copy.deepcopy(ref).to(dtype)
            gsum = [torch.zeros_like(p, dtype=torch.float32) for p in ref.parameters()]
            for q in range(n):
                shadow.zero_grad()
                F.mse_loss(shadow(X[q * 4:(q + 1) * 4].to(dtype)).float(), Y[q * 4:(q + 1) * 4]).backward()
                for a, p in zip(gsum, shadow.parameters()):
                    a += p.grad.float()
            for p, a in zip(ref.parameters(), gsum):
                p.grad = a / n
        ropt.step()
        xs, ys = X[r * 4:(r + 1) * 4], Y[r * 4:(r + 1) * 4]
        F.mse_loss(model(xs.to(dtype)).float(), ys).backward()
        opt.step()
        opt.zero_grad()
        if dtype != torch.float32:
            # keep the fp32 reference in lock-step with the bf16-rounded weights it would see
            pass
    torch.cuda.synchronize()
    tol = dict(rtol=2e-4, atol=2e-5) if dtype == torch.float32 else dict(rtol=3e-2, atol=3e-2)
    for a, b in zip(model.parameters(), ref.parameters()):
        torch.testing.assert_close(a.float(), b, **tol)
    # gradients were zeroed by the kernel
    assert all(float(p.grad.abs().max()) == 0.0 for p in model.parameters())
    flat = torch.cat([p.detach().reshape(-1).float() for p in model.parameters()])
    g = [torch.empty_like(flat) for _ in range(n)]
    dist.all_gather(g, flat)
    assert all(torch.equal(g[0], q) for q in g), "replicas diverged"
    # state export parity (momentum / exp_avg visible through state_dict)
    opt.fused_engine.export_state()
    sd = opt.state_dict()["state"]
    rsd = ropt.state_dict()["state"]
    key = "momentum_buffer" if opt_name.startswith("sgd") else "exp_avg"
    if dtype == torch.float32:
        for i in rsd:
            torch.testing.assert_close(sd[i][key].float().cpu(), rsd[i][key].cpu(), rtol=2e-4, atol=2e-5)
    s.check_errors()
    return opt.fused_engine.algorithms()


def lstm_dp_training(hvd):
    """End-to-end: reference LSTM config over the fused engine; equals the NCCL stand-in."""
    from distributed_torch_horovod_gcp_b200.models import LSTM
    s = _symm(hvd)
    r, n = hvd.rank(), hvd.size()
    dev = s.device
    torch.manual_seed(0)
    m = LSTM(23, 10, 1, 256, device=dev)
    ref = copy.deepcopy(m)
    opt = hvd.DistributedOptimizer(torch.optim.Adam(m.parameters(), lr=1e-3),
                                   named_parameters=m.named_parameters())
    ropt = torch.optim.Adam(ref.parameters(), lr=1e-3)
    hvd.broadcast_parameters(m.state_dict(), root_rank=0)
    assert opt.fused_engine is not None
    for step in range(5):
        torch.manual_seed(100 + step * n + r)
        x, y = torch.randn(32, 10, 23, device=dev), torch.randn(32, 1, 1, device=dev)
        for mod, o, is_ref in ((m, opt, False), (ref, ropt, True)):
            torch.manual_seed(7 + step * n + r)          # same random (h0,c0) for both
            F.mse_loss(mod(x), y).backward()
            if is_ref:
                for p in mod.parameters():
                    dist.all_reduce(p.grad)
                    p.grad /= n
            o.step()
            o.zero_grad()
    torch.cuda.synchronize()
    # Adam normalises by sqrt(v): last-bit differences in the cross-rank summation order
    # (fixed rank order here vs NCCL's) are amplified on near-zero gradients -> loose rtol.
    for a, b in zip(m.parameters(), ref.parameters()):
        torch.testing.assert_close(a, b, rtol=2e-2, atol=2e-5)
    s.check_errors()
    return opt.fused_engine.algorithms()


def stress_flag_reuse(hvd, iters):
    """Repeated collectives of varying size with per-iteration checksum (flag-reuse bugs)."""
    s = _symm(hvd)
    r, n = hvd.rank(), hvd.size()
    dev = s.device
    st = hvd.symm_empty(1 << 18, torch.float32)
    bad = 0
    for i in range(iters):
        numel = [256, 4096, 65536, 1 << 18][i % 4]
        v = st[:numel]
        v.fill_(float((i % 13) + r))
        hvd.allreduce_(v, op=hvd.Sum)
        want = float(sum((i % 13) + q for q in range(n)))
        if i % 50 == 0 or i == iters - 1:
            torch.cuda.synchronize()
            if not bool(torch.all(v == want)):
                bad += 1
    torch.cuda.synchronize()
    s.check_errors()
    assert bad == 0, bad
    return True


def watchdog_timeout(hvd):
    """Failure detection (SURVEY.md §5.3): a rank that never joins a collective must not hang its
    peers' GPUs — the bounded spin-wait expires, the kernel reports through the host mailbox and
    the host raises HorovodInternalError naming the straggler."""
    import time
    s = _symm(hvd)
    r = hvd.rank()
    t = hvd.symm_empty(1 << 12, torch.float32)
    t.fill_(1.0)
    hvd.allreduce_(t, op=hvd.Sum)                 # one healthy collective first
    torch.cuda.synchronize()
    s.check_errors()
    raised = False
    if r != 1:
        t0 = time.time()
        hvd.allreduce_(t, op=hvd.Sum)             # rank 1 never shows up
        torch.cuda.synchronize()
        dt = time.time() - t0
        try:
            s.check_errors()
        except hvd.HorovodInternalError as e:
            raised = "timed out waiting for rank" in str(e)
        assert raised, "watchdog did not fire"
        assert dt < 30, dt
    else:
        time.sleep(6)
    return raised or r == 1


def native_collectives_match_nccl(hvd):
    """reduce-scatter / all-gather / all-to-all on the sm_90a kernels vs torch.distributed (NCCL)."""
    s = _symm(hvd)
    r, n = hvd.rank(), hvd.size()
    dev = s.device
    launches0 = s.launches
    for dtype, tol in ((torch.float32, 1e-5), (torch.bfloat16, 2e-2)):
        for rows in (n * 8, n * 1024, n * 40000):
            torch.manual_seed(rows + r)
            x = torch.randn(rows, 16, device=dev).to(dtype)
            # reduce-scatter (Average and Sum)
            ref = x.float().clone()
            dist.all_reduce(ref)
            per = rows // n
            for op, scale in ((hvd.Sum, 1.0), (hvd.Average, 1.0 / n)):
                out = hvd.reducescatter(x, op=op)
                want = ref[r * per:(r + 1) * per] * scale
                assert out.shape == want.shape
                err = (out.float() - want).abs().max().item() / max(want.abs().max().item(), 1e-6)
                assert err < tol, ("reducescatter", dtype, rows, err)
            # all-gather
            g = hvd.allgather(x)
            refs = [torch.empty_like(x) for _ in range(n)]
            dist.all_gather(refs, x)
            assert torch.equal(g, torch.cat(refs, dim=0)), ("allgather", dtype, rows)
            # all-to-all (equal splits)
            a = hvd.alltoall(x)
            ins = list(x.chunk(n, dim=0))
            outs = [torch.empty_like(c) for c in ins]
            dist.all_to_all(outs, ins)
            assert torch.equal(a, torch.cat(outs, dim=0)), ("alltoall", dtype, rows)
    assert s.launches - launches0 >= 2 * 3 * 4, "native kernels did not run"
    # ragged all-gather keeps Horovod semantics (fallback path)
    t = torch.full((r + 1, 3), float(r), device=dev)
    g = hvd.allgather(t)
    assert g.shape[0] == n * (n + 1) // 2
    torch.cuda.synchronize()
    s.check_errors()
    return True


def sync_bn_kernel_path(hvd):
    """SyncBatchNorm on NHWC bf16: fused BN kernels + one-shot allreduce == fp32 BN over the global batch."""
    s = _symm(hvd)
    r, n = hvd.rank(), hvd.size()
    dev = s.device
    from distributed_torch_horovod_gcp_b200.ops import counters, kernels
    assert kernels.has("bn_act")
    torch.manual_seed(5)
    C = 64
    full = torch.randn(n * 4, C, 8, 8, device=dev)
    gfull = torch.randn(n * 4, C, 8, 8, device=dev)
    bn = hvd.SyncBatchNorm(C).to(dev).to(torch.bfloat16)
    with torch.no_grad():
        bn.weight.copy_(torch.rand(C) + 0.5)
        bn.bias.copy_(torch.randn(C) * 0.1)
    x = full[r * 4:(r + 1) * 4].to(torch.bfloat16).contiguous(memory_format=torch.channels_last).requires_grad_(True)
    y = bn(x)
    y.backward(gfull[r * 4:(r + 1) * 4].to(torch.bfloat16).contiguous(memory_format=torch.channels_last))
    # oracle: plain BN in fp32 over the whole batch (bf16-rounded inputs)
    ref = torch.nn.BatchNorm2d(C).to(dev)
    with torch.no_grad():
        ref.weight.copy_(bn.weight.float())
        ref.bias.copy_(bn.bias.float())
    xf = full.to(torch.bfloat16).float().requires_grad_(True)
    yr = ref(xf)
    yr.backward(gfull.to(torch.bfloat16).float())
    rel = lambda a, b: ((a.float() - b.float()).norm() / b.float().norm().clamp_min(1e-6)).item()
    assert rel(y, yr[r * 4:(r + 1) * 4]) < 1e-2
    assert rel(x.grad, xf.grad[r * 4:(r + 1) * 4]) < 2e-2
    # local parameter gradients sum (over ranks) to the global ones
    gw = hvd.allreduce(bn.weight.grad.float(), op=hvd.Sum)
    assert rel(gw, ref.weight.grad) < 2e-2
    assert rel(bn.running_var.float(), ref.running_var) < 2e-2
    s.check_errors()
    return True


def fused_engine_cuda_graph(hvd):
    """The headline path: fused engine + whole-step CUDA graph at N > 1 trains like the eager fused path."""
    from distributed_torch_horovod_gcp_b200.models import resnet18
    from distributed_torch_horovod_gcp_b200.utils.graph import GraphedStep
    s = _symm(hvd)
    r, n = hvd.rank(), hvd.size()
    dev = s.device
    losses = {}
    for mode in ("eager", "graph"):
        torch.manual_seed(0)
        m = resnet18(num_classes=10).to(dev).to(torch.bfloat16).to(memory_format=torch.channels_last)
        opt = hvd.DistributedOptimizer(torch.optim.SGD(m.parameters(), lr=0.02, momentum=0.9),
                                       named_parameters=m.named_parameters())
        hvd.broadcast_parameters(m.state_dict(), root_rank=0)
        assert opt.fused_engine is not None
        torch.manual_seed(10 + r)
        x = torch.randn(8, 3, 64, 64, device=dev).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
        y = torch.randint(0, 10, (8,), device=dev)

        def step(x, y):
            loss = F.cross_entropy(m(x).float(), y)
            loss.backward()
            opt.step()
            opt.zero_grad()
            return loss.detach()
        fn = GraphedStep(step, [x, y], warmup=2) if mode == "graph" else step
        ls = [float(fn(x, y)) for _ in range(6)]
        torch.cuda.synchronize()
        assert all(l == l for l in ls), ls
        # replicas stay bit-identical
        flat = torch.cat([p.detach().float().reshape(-1) for p in m.parameters()])
        g = [torch.empty_like(flat) for _ in range(n)]
        dist.all_gather(g, flat)
        assert all(torch.equal(g[0], q) for q in g), mode
        losses[mode] = ls
        opt.remove_hooks()
    # graph warm-up consumed 3 extra steps (2 warm-up + capture): the loss must keep decreasing
    assert losses["eager"][-1] < losses["eager"][0]
    assert losses["graph"][-1] < losses["eager"][0]
    s.check_errors()
    return losses


def model_to_after_wrap(hvd):
    """ADVICE r1 (high): `model.to(device)` AFTER DistributedOptimizer re-flattens nn.LSTM weights into a
    fresh cuDNN buffer; the engine must notice and re-home them, and the LSTM weights must train."""
    from distributed_torch_horovod_gcp_b200.models import LSTM
    s = _symm(hvd)
    r, n = hvd.rank(), hvd.size()
    dev = s.device
    torch.manual_seed(0)
    m = LSTM(23, 10, 1, 256, device=dev)
    ref = copy.deepcopy(m)
    opt = hvd.DistributedOptimizer(torch.optim.Adam(m.parameters(), lr=1e-3),
                                   named_parameters=m.named_parameters())
    m.to(dev)                                   # reference order: app/torch_train.py:259 then :261
    ropt = torch.optim.Adam(ref.parameters(), lr=1e-3)
    hvd.broadcast_parameters(m.state_dict(), root_rank=0)
    w0 = m.lstm.weight_hh_l0.detach().clone()
    for step in range(3):
        torch.manual_seed(100 + step * n + r)
        x, y = torch.randn(32, 10, 23, device=dev), torch.randn(32, 1, 1, device=dev)
        for mod, o, is_ref in ((m, opt, False), (ref, ropt, True)):
            torch.manual_seed(7 + step * n + r)
            F.mse_loss(mod(x), y).backward()
            if is_ref:
                for p in mod.parameters():
                    dist.all_reduce(p.grad)
                    p.grad /= n
            o.step()
            o.zero_grad()
    torch.cuda.synchronize()
    assert not torch.equal(m.lstm.weight_hh_l0, w0), "LSTM weights were never updated"
    for (na, a), b in zip(m.named_parameters(), ref.parameters()):
        torch.testing.assert_close(a, b, rtol=2e-2, atol=2e-5, msg=na)
    s.check_errors()
    return opt.fused_engine.rehomed


def init_shutdown_cycles(hvd):
    """init -> train -> shutdown -> init twice in one process: symmetric memory is released each time."""
    from distributed_torch_horovod_gcp_b200 import _state
    free0 = None
    for cycle in range(3):
        s = _symm(hvd)
        dev = s.device
        m = torch.nn.Linear(512, 512).to(dev)
        opt = hvd.DistributedOptimizer(torch.optim.SGD(m.parameters(), lr=0.1),
                                       named_parameters=m.named_parameters())
        assert opt.fused_engine is not None
        for _ in range(2):
            m(torch.randn(4, 512, device=dev)).sum().backward()
            opt.step()
            opt.zero_grad()
        t = torch.full((1024,), float(hvd.rank()), device=dev)
        assert float(hvd.allreduce(t, op=hvd.Sum)[0]) == sum(range(hvd.size()))
        torch.cuda.synchronize()
        s.check_errors()
        opt.remove_hooks()
        hvd.shutdown()
        assert float(m.weight.sum()) == float(m.weight.sum())       # parameters survive the release
        free, _ = torch.cuda.mem_get_info(dev)
        if free0 is None:
            free0 = free
        else:   # no 64 MiB-per-cycle staging leak (allow allocator noise)
            assert free0 - free < (48 << 20), (cycle, free0, free)
        hvd.init()
    return True


def allreduce_large(hvd):
    """256 MiB and 1 GiB fp32 buckets through every algorithm (NVLS tail path included) vs NCCL."""
    s = _symm(hvd)
    from distributed_torch_horovod_gcp_b200.runtime import symm as S
    r, n = hvd.rank(), hvd.size()
    dev = s.device
    for numel in ((64 << 20) + 4, (256 << 20) + 4):
        t = hvd.symm_empty(numel, torch.float32)
        torch.manual_seed(r)
        base = torch.randn(1 << 20, device=dev)
        t.view(-1)[: (numel // (1 << 20)) * (1 << 20)].view(-1, 1 << 20).copy_(base.expand(numel // (1 << 20), -1))
        t.view(-1)[(numel // (1 << 20)) * (1 << 20):] = 1.0
        ref = base.clone()
        dist.all_reduce(ref)
        for algo in ("twoshot", "nvls"):
            if algo == "nvls" and not s.multicast:
                continue
            code = {"twoshot": S.ALGO_TWOSHOT, "nvls": S.ALGO_NVLS}[algo]
            y = t.clone() if False else t      # in place in symmetric memory
            snap = y.view(-1)[:8].clone()
            ev = s.allreduce_(y, algo=code)
            ev.synchronize()
            got = y.view(-1)[: 1 << 20]
            err = (got - ref).abs().max().item() / ref.abs().max().item()
            assert err < 1e-5, (numel, algo, err)
            tail = y.view(-1)[-4:]
            assert torch.allclose(tail, torch.full_like(tail, float(n))), (numel, algo, tail)
            # restore the inputs for the next algorithm
            t.view(-1)[: (numel // (1 << 20)) * (1 << 20)].view(-1, 1 << 20).copy_(base.expand(numel // (1 << 20), -1))
            t.view(-1)[(numel // (1 << 20)) * (1 << 20):] = 1.0
        del t
    s.check_errors()
    return True


def compressed_engine(hvd, wire):
    """hvd.Compression.bf16 / fp16 with fp32 parameters stays on the fused engine: 16-bit gradients on the
    wire, fp32 sum + update inside the same kernel; result == torch optimizer on fp32-averaged gradients
    up to the wire rounding; replicas bit-identical."""
    s = _symm(hvd)
    r, n = hvd.rank(), hvd.size()
    dev = s.device
    comp = {"bf16": hvd.Compression.bf16, "fp16": hvd.Compression.fp16}[wire]
    torch.manual_seed(0)
    m = torch.nn.Sequential(torch.nn.Linear(300, 257), torch.nn.Tanh(), torch.nn.Linear(257, 10)).to(dev)
    ref = copy.deepcopy(m)
    opt = hvd.DistributedOptimizer(torch.optim.SGD(m.parameters(), lr=0.05, momentum=0.9),
                                   named_parameters=m.named_parameters(), compression=comp,
                                   gradient_predivide_factor=2.0)
    ropt = torch.optim.SGD(ref.parameters(), lr=0.05, momentum=0.9)
    hvd.broadcast_parameters(m.state_dict(), root_rank=0)
    eng = opt.fused_engine
    assert eng is not None and eng.wire is not None, "compression must not disable the fused engine"
    assert set(eng.algorithms().values()) == {"oneshot"}
    for step in range(4):
        torch.manual_seed(50 + step * n + r)
        x, y = torch.randn(16, 300, device=dev), torch.randint(0, 10, (16,), device=dev)
        for mod, o, is_ref in ((m, opt, False), (ref, ropt, True)):
            F.cross_entropy(mod(x), y).backward()
            if is_ref:
                for p in mod.parameters():
                    dist.all_reduce(p.grad)
                    p.grad /= n
            o.step()
            o.zero_grad()
    torch.cuda.synchronize()
    for a, b in zip(m.parameters(), ref.parameters()):
        assert a.dtype == torch.float32
        torch.testing.assert_close(a, b, rtol=3e-2, atol=3e-4)
    flat = torch.cat([p.detach().reshape(-1) for p in m.parameters()])
    g = [torch.empty_like(flat) for _ in range(n)]
    dist.all_gather(g, flat)
    assert all(torch.equal(g[0], q) for q in g)
    s.check_errors()
    return True
