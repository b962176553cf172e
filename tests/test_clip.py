"""Gradient clipping by global norm (``DistributedOptimizer(max_grad_norm=)``) on the generic path over Gloo,
and at world size 1 where the wrapper is the plain optimizer."""
import math

import pytest

from mp_util import run_workers


@pytest.mark.parametrize("world,opt", [(1, "sgd"), (2, "sgd"), (2, "adam"), (2, "adamw")])
def test_generic_clip_matches_torch(world, opt):
    res = run_workers(world, "clip_cases", "generic_matches_torch", (opt, 0.05))
    assert all(r == res[0] for r in res), "grad_norm differs across ranks"
    assert all(math.isfinite(v) and v > 0.05 for v in res[0])


@pytest.mark.parametrize("world", [1, 2])
def test_unset_is_none_and_invalid_values_raise(world):
    assert all(run_workers(world, "clip_cases", "unset_and_invalid"))


@pytest.mark.parametrize("bad", [0, -1, float("inf"), float("nan")])
def test_invalid_max_grad_norm_raises_before_setup(bad):
    import torch
    import distributed_torch_horovod_gcp_b200.torch as hvd
    with pytest.raises(ValueError, match="max_grad_norm"):
        hvd.DistributedOptimizer(torch.optim.SGD(torch.nn.Linear(2, 2).parameters(), lr=0.1), max_grad_norm=bad)
