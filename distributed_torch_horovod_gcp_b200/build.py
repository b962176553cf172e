"""In-tree native build (no torch headers; a few seconds per file).

    python -m distributed_torch_horovod_gcp_b200.build [--force] [--verbose]

Produces ``distributed_torch_horovod_gcp_b200/lib/*.so`` for sm_90a (H100):
  libb200dp_comm.so     csrc/runtime.cpp + csrc/comm_kernels.cu
  libb200dp_kernels.so  csrc/gemm_sm90.cu, conv_sm90.cu, elementwise.cu, lstm_kernels.cu, lstm_rec_sm90.cu,
                        attn_sm90.cu, xent_sm90.cu
nvcc cross-compiles without a GPU, so this also runs on the CPU dev box.
"""
from __future__ import annotations

import hashlib
import os
import shutil
import subprocess
import sys
from typing import List

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "lib")

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
    "-Xcompiler", "-fPIC", "-Xcompiler", "-Wall", "-Xcompiler", "-Wno-unused-function",
    "--expt-relaxed-constexpr",
]

TARGETS = {
    "libb200dp_comm.so": ["runtime.cpp", "comm_kernels.cu"],
    "libb200dp_kernels.so": ["gemm_sm90.cu", "conv_sm90.cu", "elementwise.cu", "lstm_kernels.cu",
                             "lstm_rec_sm90.cu", "attn_sm90.cu", "xent_sm90.cu"],
}


def _nvcc() -> str:
    for c in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if c and os.path.exists(c):
            return c
    raise RuntimeError("nvcc not found")


def _digest(paths: List[str], flags: List[str]) -> str:
    h = hashlib.sha256(" ".join(flags).encode())
    for p in paths:
        with open(p, "rb") as f:
            h.update(f.read())
    for hdr in sorted(os.listdir(CSRC)):
        if hdr.endswith((".h", ".cuh")):
            with open(os.path.join(CSRC, hdr), "rb") as f:
                h.update(f.read())
    return h.hexdigest()


def build(force: bool = False, verbose: bool = False, ptxas_info: bool = False) -> List[str]:
    """Build (or re-use) the in-tree libraries.  Serialised across processes with a file lock so
    that N ranks starting on a fresh checkout do not run nvcc into the same output file."""
    import fcntl
    os.makedirs(LIB, exist_ok=True)
    with open(os.path.join(LIB, ".build.lock"), "w") as lock:
        fcntl.flock(lock, fcntl.LOCK_EX)
        try:
            return _build_locked(force, verbose, ptxas_info)
        finally:
            fcntl.flock(lock, fcntl.LOCK_UN)


def _build_locked(force: bool, verbose: bool, ptxas_info: bool) -> List[str]:
    built = []
    nvcc = _nvcc()
    for name, srcs in TARGETS.items():
        paths = [os.path.join(CSRC, s) for s in srcs if os.path.exists(os.path.join(CSRC, s))]
        if not paths:
            continue
        out = os.path.join(LIB, name)
        flags = list(NVCC_FLAGS) + (["-Xptxas", "-v"] if ptxas_info else [])
        stamp = out + ".sha256"
        dig = _digest(paths, flags)
        if not force and os.path.exists(out) and os.path.exists(stamp) and \
                open(stamp).read().strip() == dig:
            built.append(out)
            continue
        cmd = [nvcc] + flags + ["-shared", "-o", out] + paths + ["-lcudart_static", "-ldl", "-lrt", "-lpthread"]
        if verbose:
            print(" ".join(cmd), flush=True)
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"nvcc failed for {name}:\n{r.stdout}\n{r.stderr}")
        if verbose or ptxas_info:
            sys.stderr.write(r.stderr)
        with open(stamp, "w") as f:
            f.write(dig)
        built.append(out)
    return built


if __name__ == "__main__":
    outs = build(force="--force" in sys.argv, verbose="--verbose" in sys.argv or "-v" in sys.argv,
                 ptxas_info="--ptxas" in sys.argv)
    for o in outs:
        print("built", o)
