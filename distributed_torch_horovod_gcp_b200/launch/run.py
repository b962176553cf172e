"""``horovodrun``-shaped launcher.

Reference launch forms (README.md:30, Dockerfile:17; SURVEY.md §3.1):

    horovodrun -np 4 -H localhost:4 python3 app/torch_train.py

Equivalent here:

    python -m distributed_torch_horovod_gcp_b200.launch -np 4 -H localhost:4 python3 app/torch_train.py
    bin/horovodrun -np 4 -H localhost:4 python3 app/torch_train.py       (same thing)

What it does (Horovod's Gloo launch path, rebuilt): parse ``-np`` / ``-H host:slots`` /
``--hostfile``; build the slot table (rank, local_rank, cross_rank per slot); spawn one
process per slot with the rank environment (both ``RANK/WORLD_SIZE/LOCAL_RANK/…`` and the
``HOROVOD_*`` names); multiplex stdout/stderr back with a ``[rank]<stdout>:`` prefix; and
if any worker exits non-zero, terminate all the others (failure detection — SURVEY.md
§5.3).  Remote hosts are reached over ``ssh`` like ``horovodrun``.  Horovod tuning flags
are accepted and forwarded as the same ``HOROVOD_*`` environment variables the runtime
reads (``--fusion-threshold-mb`` → bucket size, ``--timeline-filename`` → timeline,
``--stall-check-*`` → the device watchdog deadline, ``--log-level`` → the package logger,
``--autotune`` → a start-up allreduce sweep that fills the algorithm table; flags that configure
Horovod machinery which does not exist here — the polling thread, the response cache, the
two-level allreduce — are reported as ignored on stderr instead of being silently swallowed).

Elastic mode (``--host-discovery-script`` with ``--min-np`` / ``--max-np``; Horovod's elastic
launcher, restart-based): the script prints ``host:slots`` lines; the job runs on
``min(max_np, available slots)`` processes; when a worker fails, or when the workers notice through
``state.check_host_updates()`` that the discovered host set changed (they persist the committed
state and exit with code 75), the launcher re-runs discovery and relaunches the whole job, which
resumes from the persisted commit (``hvd.elastic.run``).
"""
from __future__ import annotations

import argparse
import os
import shlex
import signal
import socket
import subprocess
import sys
import threading
import time
from dataclasses import dataclass
from typing import Dict, List, Optional, Sequence, Tuple

LOCAL_NAMES = {"localhost", "127.0.0.1", "::1"}


@dataclass
class Slot:
    hostname: str
    rank: int
    local_rank: int
    cross_rank: int
    size: int
    local_size: int
    cross_size: int


def parse_hosts(hosts: str) -> List[Tuple[str, int]]:
    """``"h1:4,h2:4"`` -> ``[("h1", 4), ("h2", 4)]``; a bare host means one slot."""
    out: List[Tuple[str, int]] = []
    for item in hosts.split(","):
        item = item.strip()
        if not item:
            continue
        if ":" in item:
            h, s = item.rsplit(":", 1)
            try:
                n = int(s)
            except ValueError:
                raise ValueError(f"invalid host spec {item!r}: slots must be an integer")
            if n <= 0:
                raise ValueError(f"invalid host spec {item!r}: slots must be positive")
            out.append((h, n))
        else:
            out.append((item, 1))
    if not out:
        raise ValueError("empty host list")
    return out


def parse_hostfile(path: str) -> List[Tuple[str, int]]:
    """Lines of ``hostname slots=N`` (``#`` comments allowed)."""
    out = []
    with open(path) as f:
        for line in f:
            line = line.split("#", 1)[0].strip()
            if not line:
                continue
            parts = line.split()
            slots = 1
            for p in parts[1:]:
                if p.startswith("slots="):
                    slots = int(p.split("=", 1)[1])
            out.append((parts[0], slots))
    if not out:
        raise ValueError(f"hostfile {path} lists no hosts")
    return out


def build_slots(hosts: Sequence[Tuple[str, int]], np: int) -> List[Slot]:
    """Assign ``np`` ranks to host slots in order (Horovod's host-major assignment)."""
    total = sum(s for _, s in hosts)
    if np > total:
        raise ValueError(f"requested -np {np} processes but only {total} slots are available "
                         f"on hosts {','.join(f'{h}:{s}' for h, s in hosts)}")
    placed: List[Tuple[str, int, int]] = []   # (host, host_index, local_rank)
    r = 0
    for hi, (h, s) in enumerate(hosts):
        for lr in range(s):
            if r >= np:
                break
            placed.append((h, hi, lr))
            r += 1
    local_sizes: Dict[int, int] = {}
    for _, hi, _ in placed:
        local_sizes[hi] = local_sizes.get(hi, 0) + 1
    used_hosts = sorted(local_sizes)
    slots = []
    for rank, (h, hi, lr) in enumerate(placed):
        cross_size = sum(1 for k in used_hosts if local_sizes[k] > lr)
        cross_rank = sum(1 for k in used_hosts if k < hi and local_sizes[k] > lr)
        slots.append(Slot(h, rank, lr, cross_rank, np, local_sizes[hi], cross_size))
    return slots


def _free_port() -> int:
    with socket.socket(socket.AF_INET, socket.SOCK_STREAM) as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def make_parser() -> argparse.ArgumentParser:
    p = argparse.ArgumentParser(
        prog="horovodrun", description="H100 data-parallel launcher (horovodrun-compatible CLI)")
    p.add_argument("-v", "--version", action="store_true")
    p.add_argument("-np", "--num-proc", dest="np", type=int)
    p.add_argument("-cb", "--check-build", action="store_true")
    p.add_argument("-H", "--hosts", dest="hosts")
    p.add_argument("-hostfile", "--hostfile", dest="hostfile")
    p.add_argument("-p", "--ssh-port", dest="ssh_port", type=int)
    p.add_argument("-i", "--ssh-identity-file", dest="ssh_identity_file")
    p.add_argument("--master-port", type=int, default=None,
                   help="rendezvous TCP port (default: a free port)")
    p.add_argument("--network-interface", dest="nics")
    p.add_argument("--start-timeout", type=int, default=None)
    p.add_argument("--verbose", action="store_true")
    p.add_argument("--output-filename", dest="output_filename",
                   help="directory: per-rank stdout/stderr are also written to <dir>/rank.<r>/")
    p.add_argument("--disable-cache", action="store_true")
    p.add_argument("--gloo", action="store_true", help="accepted for parity (control plane is Gloo)")
    p.add_argument("--mpi", action="store_true", help="rejected: there is no MPI in this runtime")
    p.add_argument("--fusion-threshold-mb", type=float)
    p.add_argument("--cycle-time-ms", type=float, help="accepted; no-op (no polling thread)")
    p.add_argument("--cache-capacity", type=int, help="accepted; no-op (static bucket plan)")
    p.add_argument("--hierarchical-allreduce", action="store_true")
    p.add_argument("--autotune", action="store_true",
                   help="accepted; algorithm choice is a static size table (B200DP_ALGO overrides)")
    p.add_argument("--timeline-filename")
    p.add_argument("--timeline-mark-cycles", action="store_true")
    p.add_argument("--no-stall-check", action="store_true")
    p.add_argument("--stall-check-warning-time-seconds", type=int)
    p.add_argument("--stall-check-shutdown-time-seconds", type=int)
    p.add_argument("--log-level", choices=["TRACE", "DEBUG", "INFO", "WARNING", "ERROR", "FATAL"])
    p.add_argument("--min-np", type=int, help="elastic: fewest processes the job may run on")
    p.add_argument("--max-np", type=int, help="elastic: most processes the job may run on")
    p.add_argument("--host-discovery-script",
                   help="elastic: executable printing one 'host:slots' line per available host")
    p.add_argument("--reset-limit", type=int, default=None,
                   help="elastic: maximum number of relaunches (default 10)")
    p.add_argument("--elastic-timeout", type=int, default=None,
                   help="elastic: seconds to wait for at least --min-np slots (default 600)")
    p.add_argument("command", nargs=argparse.REMAINDER)
    return p


def _env_for(slot: Slot, master_addr: str, master_port: int, args) -> Dict[str, str]:
    e = {
        "RANK": str(slot.rank), "WORLD_SIZE": str(slot.size),
        "LOCAL_RANK": str(slot.local_rank), "LOCAL_WORLD_SIZE": str(slot.local_size),
        "GROUP_RANK": str(slot.cross_rank),
        "MASTER_ADDR": master_addr, "MASTER_PORT": str(master_port),
        "HOROVOD_RANK": str(slot.rank), "HOROVOD_SIZE": str(slot.size),
        "HOROVOD_LOCAL_RANK": str(slot.local_rank), "HOROVOD_LOCAL_SIZE": str(slot.local_size),
        "HOROVOD_CROSS_RANK": str(slot.cross_rank), "HOROVOD_CROSS_SIZE": str(slot.cross_size),
        "HOROVOD_HOSTNAME": slot.hostname, "HOROVOD_CONTROLLER": "gloo",
        "HOROVOD_CPU_OPERATIONS": "gloo",
        "HOROVOD_GLOO_RENDEZVOUS_ADDR": master_addr,
        "HOROVOD_GLOO_RENDEZVOUS_PORT": str(master_port),
        "PYTHONUNBUFFERED": "1",
    }
    if args.fusion_threshold_mb is not None:
        e["HOROVOD_FUSION_THRESHOLD"] = str(int(args.fusion_threshold_mb * 1024 * 1024))
    if args.autotune:
        e["HOROVOD_AUTOTUNE"] = "1"          # runtime/tuning.py: measured algorithm table at start-up
    if args.timeline_filename:
        e["HOROVOD_TIMELINE"] = args.timeline_filename
    if args.timeline_mark_cycles:
        e["HOROVOD_TIMELINE_MARK_CYCLES"] = "1"
    # Horovod's stall inspector == the bounded spin-wait of the sm_90a kernels (runtime/symm.py reads these)
    if args.no_stall_check:
        e["HOROVOD_STALL_CHECK_DISABLE"] = "1"
    if args.stall_check_warning_time_seconds is not None:
        e["HOROVOD_STALL_CHECK_TIME_SECONDS"] = str(args.stall_check_warning_time_seconds)
    if args.stall_check_shutdown_time_seconds is not None:
        e["HOROVOD_STALL_SHUTDOWN_TIME_SECONDS"] = str(args.stall_check_shutdown_time_seconds)
    if getattr(args, "_elastic_env", None):
        e.update(args._elastic_env)
    if args.log_level:
        e["HOROVOD_LOG_LEVEL"] = args.log_level
    if args.start_timeout is not None:
        e["HOROVOD_START_TIMEOUT"] = str(args.start_timeout)
    if args.nics:
        e["GLOO_SOCKET_IFNAME"] = args.nics.split(",")[0]
        e["NCCL_SOCKET_IFNAME"] = args.nics
    return e


def _pump(stream, prefix: str, sink, logfile):
    try:
        for raw in iter(stream.readline, b""):
            line = raw.decode(errors="replace")
            sink.write(f"{prefix}{line}" if prefix else line)
            sink.flush()
            if logfile is not None:
                logfile.write(line)
                logfile.flush()
    finally:
        stream.close()


def check_build() -> str:
    from ..runtime import lib
    import torch
    rows = [
        ("Frameworks", [("PyTorch", True)]),
        ("Controllers", [("MPI", False), ("Gloo", True)]),
        ("Tensor Operations", [
            ("sm_90a symmetric-memory kernels (P2P / NVLS)", lib.available("libb200dp_comm.so")),
            ("sm_90a wgmma compute kernels", lib.available("libb200dp_kernels.so")),
            ("NCCL (fallback only)", bool(torch.distributed.is_nccl_available())),
            ("Gloo (CPU tensors)", True), ("MPI", False)]),
    ]
    out = ["b200dp launcher build check:", ""]
    for title, items in rows:
        out.append(f"Available {title}:")
        for name, ok in items:
            out.append(f"    [{'X' if ok else ' '}] {name}")
        out.append("")
    return "\n".join(out)


RESTART_EXIT = 75     # a worker asks for a relaunch (discovered hosts changed); EX_TEMPFAIL


def discover_hosts(script: str) -> List[Tuple[str, int]]:
    """Run the host-discovery script: one ``host:slots`` (or ``host slots=N`` / bare ``host``) per line."""
    r = subprocess.run([script], capture_output=True, text=True, timeout=60)
    if r.returncode != 0:
        raise RuntimeError(f"host discovery script {script} failed ({r.returncode}): {r.stderr.strip()}")
    hosts: List[Tuple[str, int]] = []
    for line in r.stdout.splitlines():
        line = line.split("#", 1)[0].strip()
        if not line:
            continue
        if "slots=" in line:
            parts = line.split()
            hosts.append((parts[0], int(parts[1].split("=", 1)[1])))
        else:
            hosts.extend(parse_hosts(line))
    return hosts


def _warn_ignored(args):
    ignored = []
    if args.cycle_time_ms is not None:
        ignored.append("--cycle-time-ms (no polling thread: buckets launch from autograd hooks)")
    if args.cache_capacity is not None:
        ignored.append("--cache-capacity (no response cache: the bucket plan is static)")
    if args.hierarchical_allreduce:
        ignored.append("--hierarchical-allreduce (one NVSwitch domain: every peer is one hop away)")
    if args.disable_cache:
        ignored.append("--disable-cache (no response cache)")
    for i in ignored:
        print(f"[launcher] ignored: {i}", file=sys.stderr)


def launch_once(args, hosts: Sequence[Tuple[str, int]], np: int, cmd: List[str]) -> int:
    """Spawn ``np`` workers on ``hosts``, multiplex their output, kill all on the first failure."""
    slots = build_slots(hosts, np)
    all_local = all(s.hostname in LOCAL_NAMES or s.hostname == socket.gethostname() for s in slots)
    master_addr = "127.0.0.1" if all_local else slots[0].hostname
    master_port = args.master_port or _free_port()
    if args.verbose:
        print(f"[launcher] {len(slots)} processes, rendezvous {master_addr}:{master_port}",
              file=sys.stderr)

    procs: List[subprocess.Popen] = []
    threads: List[threading.Thread] = []
    logs = []
    for slot in slots:
        env_add = _env_for(slot, master_addr, master_port, args)
        is_local = slot.hostname in LOCAL_NAMES or slot.hostname == socket.gethostname()
        if is_local:
            env = dict(os.environ)
            env.update(env_add)
            popen_cmd = cmd
        else:
            exports = " ".join(f"{k}={shlex.quote(v)}" for k, v in env_add.items())
            remote = f"cd {shlex.quote(os.getcwd())} && env {exports} " + \
                     " ".join(shlex.quote(c) for c in cmd)
            ssh = ["ssh", "-o", "StrictHostKeyChecking=no", "-o", "BatchMode=yes"]
            if args.ssh_port:
                ssh += ["-p", str(args.ssh_port)]
            if args.ssh_identity_file:
                ssh += ["-i", args.ssh_identity_file]
            popen_cmd = ssh + [slot.hostname, remote]
            env = dict(os.environ)
        p = subprocess.Popen(popen_cmd, env=env, stdout=subprocess.PIPE, stderr=subprocess.PIPE,
                             start_new_session=True)
        procs.append(p)
        out_f = err_f = None
        if args.output_filename:
            d = os.path.join(args.output_filename, f"rank.{slot.rank}")
            os.makedirs(d, exist_ok=True)
            out_f, err_f = open(os.path.join(d, "stdout"), "a"), open(os.path.join(d, "stderr"), "a")
            logs += [out_f, err_f]
        pre_o = f"[{slot.rank}]<stdout>:" if len(slots) > 1 else ""
        pre_e = f"[{slot.rank}]<stderr>:" if len(slots) > 1 else ""
        for stream, prefix, sink, lf in ((p.stdout, pre_o, sys.stdout, out_f),
                                         (p.stderr, pre_e, sys.stderr, err_f)):
            t = threading.Thread(target=_pump, args=(stream, prefix, sink, lf), daemon=True)
            t.start()
            threads.append(t)

    def kill_all(sig=signal.SIGTERM):
        for p in procs:
            if p.poll() is None:
                try:
                    os.killpg(p.pid, sig)     # exact process groups we started
                except (ProcessLookupError, PermissionError):
                    pass

    def on_signal(signum, frame):
        kill_all(signal.SIGTERM)
        raise KeyboardInterrupt

    old_int = signal.signal(signal.SIGINT, on_signal)
    old_term = signal.signal(signal.SIGTERM, on_signal)
    exit_code = 0
    try:
        remaining = set(range(len(procs)))
        while remaining:
            for i in list(remaining):
                rc = procs[i].poll()
                if rc is None:
                    continue
                remaining.discard(i)
                if rc != 0 and exit_code == 0:
                    exit_code = rc if rc > 0 else 128 - rc
                    print(f"[launcher] rank {i} exited with code {rc}; terminating the other "
                          f"{len(remaining)} process(es)", file=sys.stderr)
                    kill_all(signal.SIGTERM)
                    deadline = time.time() + 10
                    while time.time() < deadline and any(p.poll() is None for p in procs):
                        time.sleep(0.1)
                    kill_all(signal.SIGKILL)
            time.sleep(0.05)
    except KeyboardInterrupt:
        exit_code = 130
        time.sleep(0.5)
        kill_all(signal.SIGKILL)
    finally:
        signal.signal(signal.SIGINT, old_int)
        signal.signal(signal.SIGTERM, old_term)
        for t in threads:
            t.join(timeout=2)
        for f in logs:
            f.close()
    return exit_code


def run(argv: Optional[Sequence[str]] = None) -> int:
    parser = make_parser()
    args = parser.parse_args(argv)
    if args.version:
        from .. import __version__
        print(__version__)
        return 0
    if args.check_build:
        print(check_build())
        return 0
    if args.mpi:
        parser.error("--mpi: this runtime has no MPI controller; use the default (Gloo) control plane")
    elastic = args.host_discovery_script is not None
    if (args.min_np is not None or args.max_np is not None) and not elastic:
        parser.error("--min-np / --max-np need --host-discovery-script (elastic mode)")
    if args.np is None and not elastic:
        parser.error("-np is required")
    if args.np is not None and args.np <= 0:
        parser.error("-np must be positive")
    cmd = list(args.command)
    if cmd and cmd[0] == "--":
        cmd = cmd[1:]
    if not cmd:
        parser.error("no command given")
    if args.hosts and args.hostfile:
        parser.error("only one of -H / --hostfile may be given")
    _warn_ignored(args)

    if not elastic:
        if args.hostfile:
            hosts = parse_hostfile(args.hostfile)
        elif args.hosts:
            hosts = parse_hosts(args.hosts)
        else:
            hosts = [("localhost", args.np)]
        try:
            build_slots(hosts, args.np)
        except ValueError as e:
            parser.error(str(e))
        return launch_once(args, hosts, args.np, cmd)

    # ------------------------------------------------------------------ elastic (restart-based)
    script = os.path.abspath(args.host_discovery_script)
    if not os.access(script, os.X_OK):
        parser.error(f"--host-discovery-script {script} is not executable")
    min_np = args.min_np or args.np or 1
    max_np = args.max_np or args.np or (1 << 30)
    if min_np > max_np:
        parser.error("--min-np must not exceed --max-np")
    reset_limit = args.reset_limit if args.reset_limit is not None else 10
    wait_s = args.elastic_timeout if args.elastic_timeout is not None else 600
    state_dir = os.environ.get("B200DP_ELASTIC_STATE_DIR") or os.path.join(
        os.getcwd(), f".b200dp_elastic_{os.getpid()}")
    os.makedirs(state_dir, exist_ok=True)
    resets = 0
    while True:
        deadline = time.time() + wait_s
        while True:
            hosts = discover_hosts(script)
            total = sum(s for _, s in hosts)
            if total >= min_np:
                break
            if time.time() > deadline:
                print(f"[launcher] elastic: only {total} slot(s) discovered, need --min-np {min_np}; giving up",
                      file=sys.stderr)
                return 1
            time.sleep(1.0)
        np = min(max_np, total)
        spec = ",".join(f"{h}:{s}" for h, s in hosts)
        args._elastic_env = {"HOROVOD_ELASTIC": "1", "B200DP_DISCOVERY_SCRIPT": script,
                             "B200DP_ELASTIC_HOSTS": spec, "B200DP_ELASTIC_STATE_DIR": state_dir,
                             "B200DP_ELASTIC_RESET": str(resets)}
        print(f"[launcher] elastic: launching {np} process(es) on {spec} (reset {resets})", file=sys.stderr)
        rc = launch_once(args, hosts, np, cmd)
        if rc == 0:
            return 0
        if rc == 130 or resets >= reset_limit:
            return rc
        resets += 1
        why = "hosts changed" if rc == RESTART_EXIT else f"a worker failed (exit {rc})"
        print(f"[launcher] elastic: {why}; re-running host discovery", file=sys.stderr)


def main():
    sys.exit(run())


if __name__ == "__main__":
    main()
