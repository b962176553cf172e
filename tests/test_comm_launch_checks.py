"""Launch checks of the communication library's C entry points, without a GPU: every rejected configuration
returns -1 and names itself in ``b200dp_comm_last_error`` before any CUDA call is made."""
import ctypes
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def comm():
    sys.path.insert(0, ROOT)
    import __graft_entry__ as g
    g.build()
    from distributed_torch_horovod_gcp_b200 import build as B
    from distributed_torch_horovod_gcp_b200.runtime import symm as S
    lib = ctypes.CDLL(os.path.join(B.LIB, "libb200dp_comm.so"))
    lib.b200dp_comm_last_error.restype = ctypes.c_char_p
    return lib, S


# size: ARArgs.n (all-reduce, clip), CollArgs.chunk (collectives, elements for reduce-scatter) or BcastArgs.nbytes
GOOD = dict(blocks=4, threads=512, rank=0, world=1, channel=1, sel=0, dtype=0, size=64)
BAD = [
    ("blocks", 0), ("blocks", 129),
    ("threads", 31), ("threads", 48), ("threads", 513),
    ("world", 9), ("world", 0), ("rank", -1), ("rank", 1), ("channel", 4), ("channel", -1),
    ("sel", 3), ("sel", -1), ("dtype", 3), ("dtype", -1),
    ("size", 6),      # not whole fp32 vectors (4 elements) nor whole 16-byte broadcast vectors
]


def _call(lib, S, entry, cfg):
    """Launch ``entry`` with the configuration ``cfg`` (``sel``: algo, phase or collective mode)."""
    ctx = S.CommCtx()
    ctx.rank, ctx.world = cfg["rank"], cfg["world"]
    b = ctypes.byref
    if entry == "allreduce":
        a = S.ARArgs()
        a.channel, a.n = cfg["channel"], cfg["size"]
        return lib.b200dp_comm_allreduce(b(ctx), b(a), cfg["sel"], cfg["dtype"], cfg["blocks"], cfg["threads"], 0)
    if entry == "clip_bucket":
        a, k = S.ARArgs(), S.ClipArgs()
        a.channel, a.n = cfg["channel"], cfg["size"]
        return lib.b200dp_comm_clip_bucket(b(ctx), b(a), b(k), cfg["sel"], cfg["dtype"], cfg["blocks"],
                                           cfg["threads"], 0)
    if entry in ("lw_bucket", "muon_bucket"):
        lw = entry == "lw_bucket"
        a, k = S.ARArgs(), S.LwArgs() if lw else S.MuonArgs()
        a.channel, a.h.kind = cfg["channel"], cfg.get("kind", S.OPT_LARS if lw else S.OPT_MUON)
        k.nchunks = cfg.get("nchunks", 1)
        return getattr(lib, f"b200dp_comm_{entry}")(b(ctx), b(a), b(k), cfg["sel"], cfg["dtype"], cfg["blocks"],
                                                    cfg["threads"], 0)
    if entry == "collective":
        a = S.CollArgs()
        a.channel, a.chunk = cfg["channel"], cfg["size"]
        return lib.b200dp_comm_collective(b(ctx), b(a), cfg["sel"], cfg["dtype"], cfg["blocks"], cfg["threads"], 0)
    a = S.BcastArgs()
    a.channel, a.nbytes = cfg["channel"], cfg["size"]
    return lib.b200dp_comm_broadcast(b(ctx), b(a), cfg["blocks"], cfg["threads"], 0)


# the selector's range: algo 0..2, phase 0..1 (Muon 0..2), collective mode 0..2; broadcast has neither selector
# nor dtype
SEL_LIMIT = {"allreduce": 3, "clip_bucket": 2, "lw_bucket": 2, "muon_bucket": 3, "collective": 3}


@pytest.mark.parametrize("entry", ["allreduce", "clip_bucket", "lw_bucket", "muon_bucket", "collective", "broadcast"])
@pytest.mark.parametrize("field,value", BAD)
def test_bad_launch_config_is_rejected(comm, entry, field, value):
    lib, S = comm
    if entry == "broadcast" and field in ("sel", "dtype"):
        pytest.skip("broadcast takes no selector or dtype")
    if entry in ("lw_bucket", "muon_bucket") and field == "size":
        pytest.skip("the layer-wise and Muon kernels walk the chunk table, not n")
    if field == "sel" and value == 3:
        value = SEL_LIMIT[entry]
    cfg = dict(GOOD, **{field: value})
    assert _call(lib, S, entry, cfg) == -1
    msg = lib.b200dp_comm_last_error().decode()
    assert msg.startswith("bad ") and "launch" in msg, msg


@pytest.mark.parametrize("entry,kind,nchunks", [
    ("lw_bucket", "OPT_SGD", 1), ("lw_bucket", "OPT_ADAM", 1), ("lw_bucket", "OPT_LARS", -1),
    ("muon_bucket", "OPT_LAMB", 1), ("muon_bucket", "OPT_MUON", -1)])
def test_chunked_buckets_reject_other_optimizers_and_negative_chunks(comm, entry, kind, nchunks):
    lib, S = comm
    cfg = dict(GOOD, kind=getattr(S, kind), nchunks=nchunks)
    assert _call(lib, S, entry, cfg) == -1
    msg = lib.b200dp_comm_last_error().decode()
    what = "layer-wise" if entry == "lw_bucket" else "muon"
    assert msg.startswith(f"bad {what} launch") and f"kind={getattr(S, kind)}" in msg, msg


@pytest.mark.parametrize("entry", ["allreduce", "clip_bucket", "collective"])
@pytest.mark.parametrize("dtype", [1, 2])
def test_sixteen_bit_sizes_must_be_whole_vectors(comm, entry, dtype):
    """bf16 and fp16 vectors hold 8 elements: 12 elements (whole fp32 vectors) are refused, for reduce-scatter
    too."""
    lib, S = comm
    cfg = dict(GOOD, dtype=dtype, size=12)
    assert _call(lib, S, entry, cfg) == -1
    msg = lib.b200dp_comm_last_error().decode()
    assert msg.startswith("bad ") and "is not a multiple of 8" in msg, msg
