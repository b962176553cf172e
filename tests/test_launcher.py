"""Launcher: host parsing, slot table, env, output prefixing, kill-all on failure
(reference README.md:30 / Dockerfile:17 launch shape; SURVEY.md §3.1, §5.3)."""
import os
import subprocess
import sys
import time

import pytest

from distributed_torch_horovod_gcp_b200.launch import parse_hosts, parse_hostfile, build_slots
from distributed_torch_horovod_gcp_b200.launch.run import make_parser, check_build

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HRUN = [sys.executable, "-m", "distributed_torch_horovod_gcp_b200.launch"]


def test_parse_hosts():
    assert parse_hosts("localhost:4") == [("localhost", 4)]
    assert parse_hosts("a:2, b:3,c") == [("a", 2), ("b", 3), ("c", 1)]
    for bad in ("a:x", "a:0", ""):
        with pytest.raises(ValueError):
            parse_hosts(bad)


def test_hostfile(tmp_path):
    f = tmp_path / "hosts"
    f.write_text("# comment\nnode1 slots=4\nnode2 slots=2  # trailing\n\nnode3\n")
    assert parse_hostfile(str(f)) == [("node1", 4), ("node2", 2), ("node3", 1)]


def test_slot_table():
    s = build_slots([("localhost", 4)], 4)
    assert [(x.rank, x.local_rank, x.cross_rank, x.local_size, x.cross_size) for x in s] == \
        [(0, 0, 0, 4, 1), (1, 1, 0, 4, 1), (2, 2, 0, 4, 1), (3, 3, 0, 4, 1)]
    s = build_slots([("a", 2), ("b", 2)], 4)
    assert [(x.hostname, x.rank, x.local_rank, x.cross_rank, x.cross_size) for x in s] == \
        [("a", 0, 0, 0, 2), ("a", 1, 1, 0, 2), ("b", 2, 0, 1, 2), ("b", 3, 1, 1, 2)]
    s = build_slots([("a", 2), ("b", 2)], 3)            # uneven: b only has local_rank 0
    assert [(x.local_size, x.cross_size) for x in s] == [(2, 2), (2, 1), (1, 2)]
    with pytest.raises(ValueError, match="only 4 slots"):
        build_slots([("a", 4)], 5)


def test_reference_command_line_parses():
    a = make_parser().parse_args(["-np", "4", "-H", "localhost:4", "python3", "app/torch_train.py"])
    assert a.np == 4 and a.hosts == "localhost:4" and a.command == ["python3", "app/torch_train.py"]
    a = make_parser().parse_args(["-np", "2", "--fusion-threshold-mb", "32", "--timeline-filename",
                                  "/tmp/t.json", "--", "python", "-c", "pass"])
    assert a.fusion_threshold_mb == 32 and a.command[-1] == "pass"
    assert "sm_90a" in check_build()


def _run(args, timeout=120):
    env = dict(os.environ, PYTHONPATH=ROOT)
    return subprocess.run(HRUN + args, cwd=ROOT, env=env, capture_output=True, text=True,
                          timeout=timeout)


def test_env_and_prefixing():
    code = ("import os;print(os.environ['RANK'],os.environ['WORLD_SIZE'],os.environ['LOCAL_RANK'],"
            "os.environ['HOROVOD_RANK'],os.environ['HOROVOD_LOCAL_SIZE'],"
            "os.environ.get('HOROVOD_FUSION_THRESHOLD'))")
    r = _run(["-np", "3", "-H", "localhost:3", "--fusion-threshold-mb", "2", sys.executable, "-c", code])
    assert r.returncode == 0, r.stderr
    lines = sorted(l for l in r.stdout.splitlines() if l)
    assert lines == [f"[{i}]<stdout>:{i} 3 {i} {i} 3 2097152" for i in range(3)]


def test_kill_all_on_failure():
    code = ("import os,sys,time\n"
            "if os.environ['RANK']=='1': sys.exit(3)\n"
            "time.sleep(120)\n")
    t0 = time.time()
    r = _run(["-np", "3", sys.executable, "-c", code], timeout=60)
    assert r.returncode == 3
    assert time.time() - t0 < 30
    assert "rank 1 exited with code 3" in r.stderr


def test_cli_errors():
    assert _run(["-np", "2"]).returncode != 0                       # no command
    assert _run(["-np", "5", "-H", "localhost:2", "true"]).returncode != 0
    assert _run(["--mpi", "-np", "1", "true"]).returncode != 0
    r = _run(["--check-build"])
    assert r.returncode == 0 and "Gloo" in r.stdout
    r = subprocess.run([os.path.join(ROOT, "bin", "horovodrun"), "-np", "1", "echo", "hi"],
                       capture_output=True, text=True, timeout=60)
    assert r.returncode == 0 and r.stdout.strip() == "hi"


def test_remote_hosts_via_ssh_and_output_files(tmp_path):
    """Non-local hosts are reached over `ssh host 'cd <cwd> && env K=V... cmd'` (a fake ssh on PATH
    executes the remote command locally); --output-filename writes per-rank logs."""
    fake = tmp_path / "bin"
    fake.mkdir()
    ssh = fake / "ssh"
    ssh.write_text("#!/usr/bin/env bash\n"
                   "# fake ssh: drop options, first non-option arg is the host, the rest is the command\n"
                   "while [[ \"$1\" == -* ]]; do if [[ \"$1\" == -o || \"$1\" == -p || \"$1\" == -i ]]; then shift; fi; shift; done\n"
                   "host=\"$1\"; shift\n"
                   "echo \"ssh-to:$host\" >&2\n"
                   "exec bash -c \"$*\"\n")
    ssh.chmod(0o755)
    env = dict(os.environ, PYTHONPATH=ROOT, PATH=f"{fake}:{os.environ['PATH']}")
    code = "import os;print('R',os.environ['RANK'],os.environ['HOROVOD_HOSTNAME'],os.environ['HOROVOD_CROSS_RANK'],os.environ['MASTER_ADDR'])"
    out_dir = tmp_path / "logs"
    r = subprocess.run(HRUN + ["-np", "3", "-H", "nodeA:2,nodeB:2", "-p", "2222", "--output-filename",
                               str(out_dir), sys.executable, "-c", code],
                       cwd=ROOT, env=env, capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, r.stderr
    lines = sorted(l for l in r.stdout.splitlines() if "R " in l)
    assert lines == ["[0]<stdout>:R 0 nodeA 0 nodeA", "[1]<stdout>:R 1 nodeA 0 nodeA",
                     "[2]<stdout>:R 2 nodeB 1 nodeA"]
    assert r.stderr.count("ssh-to:nodeA") == 2 and r.stderr.count("ssh-to:nodeB") == 1
    for rank in range(3):
        assert (out_dir / f"rank.{rank}" / "stdout").read_text().startswith(f"R {rank}")
