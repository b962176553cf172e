"""Whole-step CUDA-graph capture.

The reference workload (LSTM, batch 32, 1.48 MB of gradients) is launch- and sync-bound on a
H100 (SURVEY.md §2.6: ~0.4 us of math per step), so the H100-first answer is to capture the
complete training step — forward, backward, the fused allreduce+optimizer kernels on their side
stream, and the gradient zeroing — in ONE CUDA graph and replay it.  The comm kernels keep
their cross-rank epochs in device memory, so a replayed graph stays in lock-step with its
peers; hyper-parameters are baked at capture time (use ``engine.lr_scale`` for schedules).
"""
from __future__ import annotations

from typing import Callable, Sequence

import torch

from . import nvtx


class GraphedStep:
    """``GraphedStep(fn, example_inputs)``: ``fn(*tensors) -> loss``.  Inputs are copied into
    static buffers; the returned loss is a static tensor overwritten by each replay."""

    def __init__(self, fn: Callable, example_inputs: Sequence[torch.Tensor], warmup: int = 3):
        self.fn = fn
        self.static_in = [t.clone() for t in example_inputs]
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):            # warm-up off the default stream (allocator, cuDNN plans)
            for _ in range(warmup):
                fn(*self.static_in)
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        from ..ops import counters
        from ..parallel.fused_engine import live_engines
        count = lambda: counters.total() + sum(e.kernel_launches for e in live_engines())
        c0 = count()
        self.graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.graph):
            self.static_out = fn(*self.static_in)
        self.kernels_per_replay = count() - c0     # hand-written kernels captured in the graph
        self.replays = 0

    def __call__(self, *inputs: torch.Tensor):
        for s, t in zip(self.static_in, inputs):
            if s.shape != t.shape:
                raise ValueError("GraphedStep needs fixed input shapes; got "
                                 f"{tuple(t.shape)} vs captured {tuple(s.shape)}")
            s.copy_(t, non_blocking=True)
        with nvtx.range("graphed_step.replay"):
            self.graph.replay()
        self.replays += 1
        return self.static_out
