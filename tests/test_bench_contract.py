"""bench.py / __graft_entry__ contract checks that do not need a GPU."""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_reference_arm_reports_unavailable():
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference",
                        "--gpus", "1", "--steps", "2", "--warmup", "1"], cwd=ROOT,
                       capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, r.stderr[-1000:]
    line = json.loads(r.stdout.strip().splitlines()[-1])
    assert line["impl"] == "reference" and "unavailable" in line and "horovod" in line["unavailable"]


def test_bench_without_gpu_fails_loudly():
    import torch
    if torch.cuda.is_available():
        return
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--steps", "1"], cwd=ROOT,
                       capture_output=True, text=True, timeout=300)
    assert r.returncode != 0
    assert "needs a CUDA device" in r.stdout


def test_build_entry_point_compiles_for_sm90a():
    """`build()` must produce loadable in-tree libraries (nvcc cross-compiles without a GPU)."""
    sys.path.insert(0, ROOT)
    import __graft_entry__ as g
    g.build()
    from distributed_torch_horovod_gcp_b200 import build as B
    assert any("compute_90a" in f for f in B.NVCC_FLAGS) and "-lineinfo" in B.NVCC_FLAGS
    for name in ("libb200dp_comm.so", "libb200dp_kernels.so"):
        assert os.path.exists(os.path.join(B.LIB, name))
    out = subprocess.run(["cuobjdump", "-lelf", os.path.join(B.LIB, "libb200dp_kernels.so")],
                         capture_output=True, text=True).stdout
    assert "sm_90a" in out


def test_ctypes_struct_layouts_match_the_c_structs():
    """The Python ctypes mirrors of CommCtx / ARArgs / BcastArgs must match the compiled C layout
    (checked without a GPU: the library loads and `b200dp_comm_limits` is a pure host function)."""
    import ctypes
    sys.path.insert(0, ROOT)
    import __graft_entry__ as g
    g.build()
    from distributed_torch_horovod_gcp_b200 import build as B
    from distributed_torch_horovod_gcp_b200.runtime import symm as S
    lib = ctypes.CDLL(os.path.join(B.LIB, "libb200dp_comm.so"))
    vals = [ctypes.c_int() for _ in range(6)]
    lib.b200dp_comm_limits(*[ctypes.byref(v) for v in vals])
    got = tuple(v.value for v in vals)
    assert got == (S.MAX_RANKS, S.MAX_BLOCKS, S.NUM_CHANNELS, ctypes.sizeof(S.CommCtx),
                   ctypes.sizeof(S.ARArgs), ctypes.sizeof(S.BcastArgs)), got
    klib = ctypes.CDLL(os.path.join(B.LIB, "libb200dp_kernels.so"))
    for sym in ("b200dp_gemm_bf16", "b200dp_bn_fwd", "b200dp_bn_bwd", "b200dp_ln_fwd", "b200dp_ln_bwd",
                "b200dp_maxpool_fwd", "b200dp_maxpool_bwd", "b200dp_stem_im2col", "b200dp_head_fwd",
                "b200dp_head_bwd"):
        assert hasattr(klib, sym), sym
