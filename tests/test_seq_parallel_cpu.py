"""Sequence parallelism without a GPU: the zigzag helpers, the balance of the causal work over ranks, and the
reference path of ``sp_attention`` / ``GPT(sequence_parallel=True)`` over Gloo at world sizes 2 to 4 against
the full-sequence model."""
import os
import re
import subprocess
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TESTS = os.path.dirname(os.path.abspath(__file__))
for _p in (ROOT, TESTS):
    if _p not in sys.path:
        sys.path.insert(0, _p)

from mp_util import run_workers  # noqa: E402

from distributed_torch_horovod_gcp_b200.ops import seq_parallel as sp  # noqa: E402


@pytest.mark.parametrize("world", [1, 2, 3, 4, 8])
@pytest.mark.parametrize("S", [16, 48, 1024])
def test_zigzag_round_trip(world, S):
    if S % (2 * world):
        pytest.skip("S does not split into 2 world chunks")
    x = torch.arange(3 * S * 2).view(3, S, 2)
    shards = [sp.zigzag_shard(x, 1, r, world) for r in range(world)]
    assert all(s.shape == (3, S // world, 2) for s in shards)
    assert torch.equal(sp.zigzag_unshard(shards, 1), x)
    pos = torch.cat([sp.zigzag_positions(S, r, world) for r in range(world)])
    assert torch.equal(pos.sort().values, torch.arange(S))                 # every position exactly once
    for r in range(world):
        assert torch.equal(sp.zigzag_positions(S, r, world), shards[r][0, :, 0] // 2)


def test_zigzag_rejects_uneven():
    with pytest.raises(ValueError):
        sp.zigzag_positions(10, 0, 3)
    with pytest.raises(ValueError):
        sp.zigzag_shard(torch.zeros(2, 12), 1, 0, 4)


@pytest.mark.parametrize("world", [1, 2, 3, 4, 8])
@pytest.mark.parametrize("c", [1, 2, 5])
def test_causal_pairs_balanced(world, c):
    """Every rank visits the same number of (query tile, key tile) pairs under the causal mask, and the pairs of
    all ranks are the full sequence's: the forward kernel's query tile with global index g visits g + 1 tiles."""
    T = 2 * world * c
    tiles = [sp.zigzag_positions(T, r, world) for r in range(world)]       # global tile of each local tile
    counts = [int((t + 1).sum()) for t in tiles]
    assert len(set(counts)) == 1
    assert sum(counts) == T * (T + 1) // 2
    # the backward's key blocks: block g sees query tiles g..T-1
    assert len({int((T - t).sum()) for t in tiles}) == 1


@pytest.mark.parametrize("world", [2, 3, 4])
def test_gpt_tiny_reference_path_matches_full(world):
    S = 24 * world
    res = run_workers(world, "sp_cases", "gpt_matches_full", args=(2, S), timeout=300)
    for r in res:
        assert r["loss_err"] <= 1e-5 * max(1.0, r["loss"]), r
        assert r["grad_rel_err"] <= 1e-4, r


def test_dropout_refused_under_sequence_parallelism():
    res = run_workers(2, "sp_cases", "dropout_refused")
    assert all(r == ["op", "model"] for r in res), res


def test_script_two_steps_world_two(tmp_path):
    env = dict(os.environ, PYTHONPATH=ROOT, OMP_NUM_THREADS="2")
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK"):
        env.pop(k, None)
    cmd = [sys.executable, "-m", "distributed_torch_horovod_gcp_b200.launch", "-np", "2", "-H", "localhost:2",
           sys.executable, os.path.join(ROOT, "app", "torch_train.py"), "--model", "gpt-tiny", "--device", "cpu",
           "--sequence-parallel", "--batch-size", "2", "--seq-len", "64", "--epochs", "2", "--steps-per-epoch", "2"]
    r = subprocess.run(cmd, cwd=str(tmp_path), env=env, capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr[-3000:]
    assert len(re.findall(r"\[0\]<stdout>:epoch: 0, train_loss: [\d.]+", r.stdout)) == 1, r.stdout[-2000:]
    assert re.search(r"\[0\]<stdout>:epoch: 0, test_loss: [\d.]+", r.stdout)


@pytest.mark.parametrize("flags", [["--model", "resnet18"], ["--dropout", "0.1"], ["--cuda-graph"]])
def test_script_refuses_unsupported_combinations(flags):
    sys.path.insert(0, os.path.join(ROOT, "app"))
    import torch_train
    argv = ["--model", "gpt-tiny", "--sequence-parallel"] + flags
    with pytest.raises(SystemExit):
        torch_train.parse_args(argv)
