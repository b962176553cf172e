"""Sequence-parallel groups without a GPU: ``GPT(sequence_parallel_size=G)`` over Gloo on the reference path against
one full-sequence model on every group's batch, its refusals, the training script's ``--sequence-parallel-size``,
and the group collectives' host-side check of the member list."""
import ctypes
import os
import re
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TESTS = os.path.dirname(os.path.abspath(__file__))
for _p in (ROOT, TESTS):
    if _p not in sys.path:
        sys.path.insert(0, _p)

from mp_util import run_workers  # noqa: E402


@pytest.mark.parametrize("world,G", [(4, 2), (4, 1), (3, 3)])
def test_gpt_tiny_groups_match_full(world, G):
    """Each rank's loss is the mean over its own tokens and its gradient includes the other members' queries'
    contributions through its keys and values, so the world average of the gradients is the full-sequence gradient
    over every group's batch: the optimizer needs nothing group-specific."""
    res = run_workers(world, "sp_group_cases", "gpt_groups_match_full", args=(2, 24 * G, G), timeout=300)
    for r in res:
        assert r["group_loss_err"] <= 1e-5 * max(1.0, r["group_loss"]), r
        assert r["loss_err"] <= 1e-5 * max(1.0, r["loss"]), r
        assert r["grad_rel_err"] <= 1e-4, r
    # different groups trained on different tokens
    assert len({round(r["group_loss"], 6) for r in res}) == world // G


def test_whole_world_group_is_bitwise_the_default():
    assert all(run_workers(4, "sp_group_cases", "gpt_whole_world_size_is_default", args=(2, 48), timeout=300))


def test_group_refusals():
    res = run_workers(4, "sp_group_cases", "refusals", timeout=300)
    want = ["not a divisor", "zero", "negative", "without sequence_parallel", "dropout", "attention dropout"]
    assert all(r == want for r in res), res


def test_group_sets_are_reused():
    """A second model with the same group size takes the registered sets instead of creating new groups."""
    res = run_workers(4, "sp_group_cases", "group_sets_reused", args=(2,), timeout=300)
    assert [r["ranks"] for r in res] == [[0, 1], [0, 1], [2, 3], [2, 3]], res
    assert all(r["added"] >= 2 and r["again"] == 0 and r["same"] for r in res), res


def _parse(argv, world, monkeypatch):
    sys.path.insert(0, os.path.join(ROOT, "app"))
    import torch_train
    for k in ("HOROVOD_SIZE", "OMPI_COMM_WORLD_SIZE", "PMI_SIZE"):
        monkeypatch.delenv(k, raising=False)
    monkeypatch.setenv("WORLD_SIZE", str(world))
    return torch_train.parse_args(["--model", "gpt-tiny"] + argv)


@pytest.mark.parametrize("flags", [
    ["--sequence-parallel-size", "2"],                                          # without --sequence-parallel
    ["--sequence-parallel", "--sequence-parallel-size", "3"],                   # does not divide 4
    ["--sequence-parallel", "--sequence-parallel-size", "0"],
    ["--sequence-parallel", "--sequence-parallel-size", "2", "--dropout", "0.1"],
    ["--sequence-parallel", "--sequence-parallel-size", "2", "--cuda-graph"],
    ["--sequence-parallel", "--sequence-parallel-size", "2", "--model", "resnet18"],
])
def test_script_refuses_bad_group_sizes(flags, monkeypatch):
    with pytest.raises(SystemExit):
        _parse(flags, 4, monkeypatch)


def test_script_group_size_from_flag_and_env(monkeypatch):
    assert _parse(["--sequence-parallel", "--sequence-parallel-size", "2"], 4, monkeypatch).sequence_parallel_size == 2
    assert _parse(["--sequence-parallel"], 4, monkeypatch).sequence_parallel_size is None
    monkeypatch.setenv("B200DP_SEQUENCE_PARALLEL_SIZE", "4")
    assert _parse(["--sequence-parallel"], 8, monkeypatch).sequence_parallel_size == 4


def test_script_two_epochs_world_four_groups_of_two(tmp_path):
    env = dict(os.environ, PYTHONPATH=ROOT, OMP_NUM_THREADS="1")
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK", "B200DP_SEQUENCE_PARALLEL_SIZE"):
        env.pop(k, None)
    cmd = [sys.executable, "-m", "distributed_torch_horovod_gcp_b200.launch", "-np", "4", "-H", "localhost:4",
           sys.executable, os.path.join(ROOT, "app", "torch_train.py"), "--model", "gpt-tiny", "--device", "cpu",
           "--sequence-parallel", "--sequence-parallel-size", "2", "--batch-size", "2", "--seq-len", "64",
           "--epochs", "8", "--steps-per-epoch", "2"]
    r = subprocess.run(cmd, cwd=str(tmp_path), env=env, capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr[-3000:]
    for e in (0, 1):
        assert len(re.findall(rf"\[0\]<stdout>:epoch: {e}, train_loss: [\d.]+", r.stdout)) == 1, r.stdout[-2000:]
        assert re.search(rf"\[0\]<stdout>:epoch: {e}, test_loss: [\d.]+", r.stdout), r.stdout[-2000:]
    assert not re.search(r"epoch: 2,", r.stdout)


# ------------------------------------------------------------------ host check of the member list
@pytest.fixture(scope="module")
def comm():
    import __graft_entry__ as g
    g.build()
    from distributed_torch_horovod_gcp_b200 import build as B
    from distributed_torch_horovod_gcp_b200.runtime import symm as S
    lib = ctypes.CDLL(os.path.join(B.LIB, "libb200dp_comm.so"))
    lib.b200dp_comm_last_error.restype = ctypes.c_char_p
    assert lib.b200dp_comm_group_coll_bytes() == ctypes.sizeof(S.GroupCollArgs)
    return lib, S


# world 8, caller world rank 3; (members, index, what the message names)
BAD_GROUPS = [
    ([2, 3, 3], 1, "strictly ascending"),           # duplicate
    ([3, 2], 0, "strictly ascending"),              # unsorted
    ([3, 8], 0, "outside the world"),
    ([-1, 3], 1, "outside the world"),
    ([0, 1], 0, "members[index]"),                  # without the caller
    ([1, 3], 0, "members[index]"),                  # index is not the caller's
    ([3, 5], 2, "members[index]"),                  # index past the group
    ([], 0, "size"),
    (list(range(9)), 3, "size"),                    # more than 8 members
]


@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("members,index,why", BAD_GROUPS)
def test_bad_member_list_is_rejected(comm, members, index, why, mode):
    """The check runs before any CUDA call: the error is returned on a machine without a GPU too."""
    lib, S = comm
    ctx = S.CommCtx()
    ctx.rank, ctx.world = 3, 8
    a = S.group_coll_args(members[:S.MAX_RANKS], index, [], [], 64)
    a.size = len(members)
    b = ctypes.byref
    assert lib.b200dp_comm_group_collective(b(ctx), b(a), mode, 0, 4, 512, 0) == -1
    msg = lib.b200dp_comm_last_error().decode()
    assert msg.startswith("bad group collective launch") and why in msg, msg


@pytest.mark.parametrize("field,value", [("mode", 2), ("use_mc", 1), ("chunk", 6), ("blocks", 0), ("channel", 4)])
def test_bad_group_launch_is_rejected(comm, field, value):
    """All-to-all has no group form, multicast is never used, and the world launch checks apply."""
    lib, S = comm
    ctx = S.CommCtx()
    ctx.rank, ctx.world = 3, 8
    cfg = dict(dict(mode=0, use_mc=0, chunk=64, blocks=4, channel=1), **{field: value})
    a = S.group_coll_args([2, 3], 1, [], [], cfg["chunk"], channel=cfg["channel"])
    a.coll.use_mc = cfg["use_mc"]
    b = ctypes.byref
    assert lib.b200dp_comm_group_collective(b(ctx), b(a), cfg["mode"], 0, cfg["blocks"], 512, 0) == -1
    msg = lib.b200dp_comm_last_error().decode()
    assert msg.startswith("bad group collective launch"), msg
