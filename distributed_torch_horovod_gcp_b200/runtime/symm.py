"""Python driver of the C++ symmetric-memory runtime (csrc/runtime.cpp) and of the sm_90a
communication kernels (csrc/comm_kernels.cu).

One ``SymmRuntime`` per process (= per GPU).  ``alloc`` is a *collective*: every rank creates
a cuMem allocation, the POSIX fds are exchanged over abstract unix sockets (SCM_RIGHTS), all
peers are mapped into the local VA space and — if the fabric supports NVLS — the pages are
bound to one multicast object.  The result is a ``SymmBuffer`` carrying the local pointer,
the per-peer pointers and the multicast pointer that the kernels take.

Replaces Horovod's NCCL communicator + fusion-buffer ownership (SURVEY.md §2.2 N5/N7/N8,
§5.8 item 1).  The Gloo CPU group of ``_state`` is used for rendezvous only.
"""
from __future__ import annotations

import ctypes
import os
import uuid
from typing import Dict, List, Optional, Tuple

import torch
import torch.distributed as dist

from . import lib as _lib

MAX_RANKS, MAX_BLOCKS, NUM_CHANNELS = 8, 128, 4
CH_ENGINE, CH_USER, CH_BCAST, CH_OPT = 0, 1, 2, 3
ALGO_ONESHOT, ALGO_TWOSHOT, ALGO_NVLS = 0, 1, 2
ALGO_NAMES = {0: "oneshot", 1: "twoshot", 2: "nvls"}
_DTYPE_CODE = {torch.float32: 0, torch.bfloat16: 1, torch.float16: 2}
OPT_NONE, OPT_SGD, OPT_ADAM, OPT_LARS, OPT_LAMB, OPT_MUON = 0, 1, 2, 3, 4, 5


class CommCtx(ctypes.Structure):
    _fields_ = [("sig", ctypes.c_uint64 * MAX_RANKS), ("epoch", ctypes.c_uint64),
                ("err", ctypes.c_uint64), ("timeout_ns", ctypes.c_uint64),
                ("rank", ctypes.c_int), ("world", ctypes.c_int)]


class OptHyper(ctypes.Structure):
    _fields_ = [("kind", ctypes.c_int), ("nesterov", ctypes.c_int), ("adamw", ctypes.c_int),
                ("maximize", ctypes.c_int), ("lr", ctypes.c_float), ("momentum", ctypes.c_float),
                ("dampening", ctypes.c_float), ("weight_decay", ctypes.c_float),
                ("beta1", ctypes.c_float), ("beta2", ctypes.c_float), ("eps", ctypes.c_float),
                ("pad_", ctypes.c_float)]


class ARArgs(ctypes.Structure):
    _fields_ = [("inp", ctypes.c_uint64 * MAX_RANKS), ("out", ctypes.c_uint64 * MAX_RANKS),
                ("in_mc", ctypes.c_uint64), ("out_mc", ctypes.c_uint64),
                ("master", ctypes.c_uint64), ("s0", ctypes.c_uint64), ("s1", ctypes.c_uint64),
                ("step_ctr", ctypes.c_uint64), ("ticket", ctypes.c_uint64),
                ("lr_scale", ctypes.c_uint64), ("scratch", ctypes.c_uint64),
                ("n", ctypes.c_uint64), ("scale", ctypes.c_float), ("channel", ctypes.c_int),
                ("zero_input", ctypes.c_int), ("copy_back", ctypes.c_int), ("h", OptHyper)]


class ClipArgs(ctypes.Structure):
    _fields_ = [("r", ctypes.c_uint64), ("slots", ctypes.c_uint64), ("norm", ctypes.c_uint64),
                ("coef", ctypes.c_uint64), ("max_norm", ctypes.c_float), ("nslots", ctypes.c_int)]


CLIP_REDUCE, CLIP_APPLY = 0, 1


class LwChunk(ctypes.Structure):
    _fields_ = [("first_vec", ctypes.c_int), ("nvec", ctypes.c_int), ("tfirst", ctypes.c_int),
                ("tcount", ctypes.c_int)]


class ChunkArgs(ctypes.Structure):
    _fields_ = [("r", ctypes.c_uint64), ("part", ctypes.c_uint64), ("chunks", ctypes.c_uint64),
                ("nchunks", ctypes.c_int), ("pad_", ctypes.c_int)]


class LwArgs(ctypes.Structure):
    _anonymous_ = ("tab",)          # k.r, k.part, k.chunks, k.nchunks reach the embedded ChunkArgs
    _fields_ = [("tab", ChunkArgs), ("ratio", ctypes.c_uint64), ("adaptive", ctypes.c_int),
                ("trust_coef", ctypes.c_float)]


LW_REDUCE, LW_APPLY = 0, 1


class MuonMat(ctypes.Structure):
    _fields_ = [("rows", ctypes.c_int), ("cols", ctypes.c_int), ("elem0", ctypes.c_int), ("x0", ctypes.c_int)]


class MuonArgs(ctypes.Structure):
    _anonymous_ = ("tab",)
    _fields_ = [("tab", ChunkArgs), ("mats", ctypes.c_uint64), ("x0", ctypes.c_uint64), ("o", ctypes.c_uint64),
                ("nesterov", ctypes.c_int), ("lr_mode", ctypes.c_int), ("eps", ctypes.c_float), ("pad_", ctypes.c_int)]


MUON_REDUCE, MUON_NORMALIZE, MUON_APPLY = 0, 1, 2


class BcastArgs(ctypes.Structure):
    _fields_ = [("buf", ctypes.c_uint64 * MAX_RANKS), ("buf_mc", ctypes.c_uint64),
                ("nbytes", ctypes.c_uint64), ("root", ctypes.c_int), ("channel", ctypes.c_int),
                ("use_mc", ctypes.c_int), ("pad_", ctypes.c_int)]


class CollArgs(ctypes.Structure):
    _fields_ = [("src", ctypes.c_uint64 * MAX_RANKS), ("dst", ctypes.c_uint64 * MAX_RANKS),
                ("src_mc", ctypes.c_uint64), ("dst_mc", ctypes.c_uint64), ("chunk", ctypes.c_uint64),
                ("scale", ctypes.c_float), ("channel", ctypes.c_int), ("use_mc", ctypes.c_int),
                ("pad_", ctypes.c_int)]


COLL_REDUCE_SCATTER, COLL_ALLGATHER, COLL_ALLTOALL = 0, 1, 2


class GroupCollArgs(ctypes.Structure):
    _fields_ = [("coll", CollArgs), ("members", ctypes.c_int * MAX_RANKS), ("size", ctypes.c_int),
                ("index", ctypes.c_int)]


def group_coll_args(members, index: int, src, dst, chunk: int, scale: float = 1.0,
                    channel: int = CH_USER) -> GroupCollArgs:
    """Argument block of a group reduce-scatter or all-gather (``b200dp_comm_group_collective``).  ``members``:
    the group's world ranks, ascending; ``index``: the caller's group rank; ``src`` / ``dst``: device pointers
    indexed by group rank (0 where the kernel does not read them); ``chunk`` as in ``CollArgs`` (elements for
    reduce-scatter, 16-byte vectors for all-gather).  Multicast stays off."""
    a = GroupCollArgs()
    for g, p in enumerate(src):
        a.coll.src[g] = p
    for g, p in enumerate(dst):
        a.coll.dst[g] = p
    a.coll.chunk, a.coll.scale, a.coll.channel = chunk, float(scale), channel
    for g, w in enumerate(members):
        a.members[g] = w
    a.size, a.index = len(members), index
    return a


class _Raw:
    """Expose a raw device range through ``__cuda_array_interface__`` (zero-copy into torch)."""

    def __init__(self, ptr: int, nbytes: int, owner):
        self.__cuda_array_interface__ = {"shape": (nbytes,), "typestr": "|u1",
                                         "data": (ptr, False), "version": 3, "strides": None}
        self._owner = owner


class SymmBuffer:
    def __init__(self, rt: "SymmRuntime", nbytes: int, padded: int, local_ptr: int,
                 peer_ptrs: List[int], mc_ptr: int, handles):
        self.rt, self.nbytes, self.padded = rt, nbytes, padded
        self.local_ptr, self.peer_ptrs, self.mc_ptr = local_ptr, peer_ptrs, mc_ptr
        self._handles = handles
        self._bytes = torch.as_tensor(_Raw(local_ptr, padded, self), device=rt.device)

    def tensor(self, dtype: torch.dtype, numel: Optional[int] = None, byte_offset: int = 0):
        es = torch.empty((), dtype=dtype).element_size()
        if numel is None:
            numel = (self.nbytes - byte_offset) // es
        return self._bytes[byte_offset: byte_offset + numel * es].view(dtype)

    def contains(self, ptr: int, nbytes: int) -> bool:
        return self.local_ptr <= ptr and ptr + nbytes <= self.local_ptr + self.padded

    def ptrs_at(self, byte_offset: int) -> List[int]:
        return [p + byte_offset for p in self.peer_ptrs]


def watchdog_seconds() -> float:
    """Deadline of the in-kernel bounded spin-wait (Horovod's stall inspector, on the device).
    ``B200DP_KERNEL_TIMEOUT_S`` wins; otherwise Horovod's knobs are honoured:
    ``HOROVOD_STALL_SHUTDOWN_TIME_SECONDS`` (``--stall-check-shutdown-time-seconds``), else
    ``HOROVOD_STALL_CHECK_TIME_SECONDS`` (``--stall-check-warning-time-seconds``: there is no separate
    warning phase on the device, the deadline is the warning time); ``HOROVOD_STALL_CHECK_DISABLE=1``
    (``--no-stall-check``) disables it (one week).  Default 300 s — NCCL-like minutes, so that a rank
    that is merely slow (checkpointing, data stall) does not abort a healthy job."""
    v = os.environ.get("B200DP_KERNEL_TIMEOUT_S")
    if v:
        return float(v)
    if os.environ.get("HOROVOD_STALL_CHECK_DISABLE", "0") == "1":
        return 7 * 24 * 3600.0
    for k in ("HOROVOD_STALL_SHUTDOWN_TIME_SECONDS", "HOROVOD_STALL_CHECK_TIME_SECONDS"):
        v = os.environ.get(k)
        if v and float(v) > 0:
            return float(v)
    return 300.0


class KernelLauncher:
    """The fused-kernel launches, shared by ``SymmRuntime`` and the world-size-1 ``LocalRuntime``: both provide
    ``lib``, ``ctx``, ``launches`` and ``pick_blocks``."""

    def _launched(self, rc: int):
        """Raise the library's message if a C entry point failed; count the launch otherwise."""
        if rc != 0:
            raise RuntimeError((self.lib.b200dp_comm_last_error() or b"").decode())
        self.launches += 1

    def launch_allreduce(self, args: ARArgs, algo: int, dtype: torch.dtype, nbytes: int,
                         stream: torch.cuda.Stream, blocks: Optional[int] = None):
        blocks = blocks or self.pick_blocks(algo, nbytes)
        self._launched(self.lib.b200dp_comm_allreduce(ctypes.byref(self.ctx), ctypes.byref(args), algo,
                                                      _DTYPE_CODE[dtype], blocks, 512, stream.cuda_stream))

    def launch_bucket(self, mode: str, args: ARArgs, k, phase: int, dtype: torch.dtype, nbytes: int,
                      stream: torch.cuda.Stream):
        """One phase of a bucket of the engine modes that split the bucket kernel, through the C entry point
        ``b200dp_comm_<mode>_bucket``: ``mode`` "clip" with ``ClipArgs`` ``k`` (``CLIP_REDUCE`` / ``CLIP_APPLY``),
        "lw" with ``LwArgs`` (LARS / LAMB: ``LW_REDUCE`` / ``LW_APPLY``) or "muon" with ``MuonArgs``
        (``MUON_REDUCE`` / ``MUON_NORMALIZE`` / ``MUON_APPLY``).  Every phase of a bucket runs on the same one-shot
        grid, so the clip reduce phase fills the same norm slots every step."""
        entry = getattr(self.lib, f"b200dp_comm_{mode}_bucket")
        blocks = self.pick_blocks(ALGO_ONESHOT, nbytes)
        self._launched(entry(ctypes.byref(self.ctx), ctypes.byref(args), ctypes.byref(k), phase, _DTYPE_CODE[dtype],
                             blocks, 512, stream.cuda_stream))

    def launch_clip_finalize(self, clip: ClipArgs, stream: torch.cuda.Stream):
        """Sum every bucket's norm slots (fixed order) into the global norm and the clip coefficient."""
        self._launched(self.lib.b200dp_comm_clip_finalize(ctypes.byref(clip), stream.cuda_stream))


class SymmRuntime(KernelLauncher):
    def __init__(self):
        raise RuntimeError("use SymmRuntime.create")

    # ------------------------------------------------------------------ creation
    @classmethod
    def create(cls, state) -> "SymmRuntime":
        self = object.__new__(cls)
        self.lib = _lib.load_comm()
        if self.lib is None:
            raise RuntimeError("libb200dp_comm.so is not built")
        self._bind()
        self.rank, self.world = state.rank, state.size
        self.group = state.cpu_group
        if state.local_size != state.size:
            raise RuntimeError("symmetric runtime spans one NVSwitch domain (single host) only")
        if self.world > MAX_RANKS:
            raise RuntimeError(f"world size {self.world} > {MAX_RANKS}")
        self.dev_index = torch.cuda.current_device()
        self.device = torch.device("cuda", self.dev_index)
        self._ck(self.lib.b200dp_rt_init(self.dev_index))
        caps = (ctypes.c_int * 8)()
        gran, mcg = ctypes.c_size_t(0), ctypes.c_size_t(0)
        self._ck(self.lib.b200dp_rt_caps(self.dev_index, caps, ctypes.byref(gran),
                                         ctypes.byref(mcg), self.world))
        if not (caps[0] and caps[1]):
            raise RuntimeError("device lacks VMM / POSIX-fd shareable handles")
        self.sm_count, self.cc = caps[3], (caps[4], caps[5])
        self.gran = max(int(gran.value), 1 << 21)
        mc_ok = bool(caps[2]) and os.environ.get("B200DP_DISABLE_NVLS", "0") != "1"
        # every rank must agree on multicast availability and device ids must be distinct
        info = [None] * self.world
        dist.all_gather_object(info, (self.dev_index, mc_ok, int(mcg.value), os.getpid()),
                               group=self.group)
        if len({i[0] for i in info}) != self.world:
            raise RuntimeError(f"ranks share CUDA devices: {[i[0] for i in info]}")
        self.peer_devs = [i[0] for i in info]
        self.multicast = all(i[1] for i in info)
        self.mc_gran = max([i[2] for i in info] + [0]) if self.multicast else 0
        for d in self.peer_devs:
            if d != self.dev_index and not self.lib.b200dp_can_access_peer(self.dev_index, d):
                raise RuntimeError(f"no P2P access {self.dev_index}->{d}")
        job = [uuid.uuid4().hex[:12] if self.rank == 0 else None]
        dist.broadcast_object_list(job, src=0, group=self.group)
        self.job = job[0]
        self._sock = self.lib.b200dp_fd_listen(self._sock_name(self.rank).encode())
        if self._sock < 0:
            raise RuntimeError("fd_listen: " + self._err())
        dist.barrier(group=self.group)
        self._alloc_id = 0
        self._pending_fds: Dict[Tuple[int, int], int] = {}
        self.buffers: List[SymmBuffer] = []
        self.timeout_ms = int(os.environ.get("B200DP_FD_TIMEOUT_MS", "60000"))

        # signal pad + epoch counters + error mailbox
        sig_bytes = NUM_CHANNELS * MAX_BLOCKS * MAX_RANKS * 4
        self.sig = self.alloc(sig_bytes, multicast=False)
        self.sig.tensor(torch.int32).zero_()
        self.epoch = torch.zeros(NUM_CHANNELS * MAX_BLOCKS * MAX_RANKS, dtype=torch.int32,
                                 device=self.device)
        hp, dp = ctypes.c_uint64(0), ctypes.c_uint64(0)
        self._ck(self.lib.b200dp_host_mailbox(64, ctypes.byref(hp), ctypes.byref(dp)))
        self._mailbox = (ctypes.c_int * 16).from_address(hp.value)
        self.ctx = CommCtx()
        for r in range(self.world):
            self.ctx.sig[r] = self.sig.peer_ptrs[r]
        self.ctx.epoch = self.epoch.data_ptr()
        self.ctx.err = dp.value
        self.ctx.timeout_ns = int(watchdog_seconds() * 1e9)
        self.ctx.rank, self.ctx.world = self.rank, self.world
        torch.cuda.synchronize(self.device)
        dist.barrier(group=self.group)

        # staging for tensors that do not live in symmetric memory
        self.stage_bytes = int(os.environ.get("B200DP_STAGING_BYTES", str(64 << 20)))
        self.stage = self.alloc(self.stage_bytes)
        self.max_blocks = int(os.environ.get("B200DP_COMM_BLOCKS", "0"))
        self.algo_override = os.environ.get("B200DP_ALGO", "auto").lower()
        self.launches = 0
        return self

    def _bind(self):
        L = self.lib
        L.b200dp_last_error.restype = ctypes.c_char_p
        L.b200dp_comm_last_error.restype = ctypes.c_char_p
        u64, i, sz = ctypes.c_uint64, ctypes.c_int, ctypes.c_size_t
        P = ctypes.POINTER
        L.b200dp_rt_init.argtypes = [i]
        L.b200dp_rt_caps.argtypes = [i, P(i), P(sz), P(sz), i]
        L.b200dp_mem_create.argtypes = [i, sz, P(u64), P(i)]
        L.b200dp_mem_import.argtypes = [i, P(u64)]
        L.b200dp_mem_map.argtypes = [i, u64, sz, sz, P(u64)]
        L.b200dp_mem_unmap.argtypes = [u64, sz]
        L.b200dp_mem_release.argtypes = [u64]
        L.b200dp_mc_create.argtypes = [i, sz, P(u64), P(i)]
        L.b200dp_mc_add_device.argtypes = [u64, i]
        L.b200dp_mc_bind.argtypes = [u64, sz, u64, sz, sz]
        L.b200dp_mc_unbind.argtypes = [u64, i, sz, sz]
        L.b200dp_fd_listen.argtypes = [ctypes.c_char_p]
        L.b200dp_fd_send.argtypes = [ctypes.c_char_p, i, i, i, i]
        L.b200dp_fd_recv.argtypes = [i, P(i), P(i), i]
        L.b200dp_fd_close.argtypes = [i]
        L.b200dp_host_mailbox.argtypes = [sz, P(u64), P(u64)]
        L.b200dp_can_access_peer.argtypes = [i, i]
        L.b200dp_comm_allreduce.argtypes = [P(CommCtx), P(ARArgs), i, i, i, i, u64]
        L.b200dp_comm_broadcast.argtypes = [P(CommCtx), P(BcastArgs), i, i, u64]
        L.b200dp_comm_clip_bucket.argtypes = [P(CommCtx), P(ARArgs), P(ClipArgs), i, i, i, i, u64]
        L.b200dp_comm_clip_finalize.argtypes = [P(ClipArgs), u64]
        L.b200dp_comm_lw_bucket.argtypes = [P(CommCtx), P(ARArgs), P(LwArgs), i, i, i, i, u64]
        L.b200dp_comm_muon_bucket.argtypes = [P(CommCtx), P(ARArgs), P(MuonArgs), i, i, i, i, u64]
        if hasattr(L, "b200dp_comm_collective"):
            L.b200dp_comm_collective.argtypes = [P(CommCtx), P(CollArgs), i, i, i, i, u64]
            if L.b200dp_comm_coll_bytes() != ctypes.sizeof(CollArgs):
                raise RuntimeError("ctypes/C struct layout mismatch: CollArgs")
            L.b200dp_comm_group_collective.argtypes = [P(CommCtx), P(GroupCollArgs), i, i, i, i, u64]
            if L.b200dp_comm_group_coll_bytes() != ctypes.sizeof(GroupCollArgs):
                raise RuntimeError("ctypes/C struct layout mismatch: GroupCollArgs")
        lim = [ctypes.c_int() for _ in range(6)]
        L.b200dp_comm_limits(*[ctypes.byref(x) for x in lim])
        got = tuple(x.value for x in lim) + (L.b200dp_comm_clip_bytes(), L.b200dp_comm_lw_bytes(),
                                             L.b200dp_comm_muon_bytes())
        want = (MAX_RANKS, MAX_BLOCKS, NUM_CHANNELS, ctypes.sizeof(CommCtx), ctypes.sizeof(ARArgs),
                ctypes.sizeof(BcastArgs), ctypes.sizeof(ClipArgs), ctypes.sizeof(LwArgs), ctypes.sizeof(MuonArgs))
        if got != want:
            raise RuntimeError(f"ctypes/C struct layout mismatch: C={got} python={want}")

    def _err(self) -> str:
        return (self.lib.b200dp_last_error() or b"").decode(errors="replace")

    def _ck(self, rc: int):
        if rc != 0:
            raise RuntimeError(self._err())

    def _sock_name(self, r: int) -> str:
        return f"b200dp-{self.job}-{r}"

    # ------------------------------------------------------------------ fd exchange
    def _send_fd(self, dst: int, fd: int, tag: int):
        rc = self.lib.b200dp_fd_send(self._sock_name(dst).encode(), fd, self.rank, tag,
                                     self.timeout_ms)
        if rc != 0:
            raise RuntimeError("fd_send: " + self._err())

    def _recv_fd(self, src: int, tag: int) -> int:
        key = (src, tag)
        while key not in self._pending_fds:
            s, t = ctypes.c_int(-1), ctypes.c_int(-1)
            fd = self.lib.b200dp_fd_recv(self._sock, ctypes.byref(s), ctypes.byref(t),
                                         self.timeout_ms)
            if fd < 0:
                raise RuntimeError("fd_recv: " + self._err())
            self._pending_fds[(s.value, t.value)] = fd
        return self._pending_fds.pop(key)

    # ------------------------------------------------------------------ allocation (collective)
    def alloc(self, nbytes: int, multicast: bool = True) -> SymmBuffer:
        use_mc = multicast and self.multicast
        g = max(self.gran, self.mc_gran if use_mc else 0)
        padded = (max(nbytes, 1) + g - 1) // g * g
        aid = self._alloc_id
        self._alloc_id += 1
        tag, mtag = 2 * aid, 2 * aid + 1
        h, fd = ctypes.c_uint64(0), ctypes.c_int(-1)
        self._ck(self.lib.b200dp_mem_create(self.dev_index, padded, ctypes.byref(h),
                                            ctypes.byref(fd)))
        for r in range(self.world):
            if r != self.rank:
                self._send_fd(r, fd.value, tag)
        handles = {self.rank: h.value}
        for r in range(self.world):
            if r != self.rank:
                pfd = self._recv_fd(r, tag)
                ph = ctypes.c_uint64(0)
                self._ck(self.lib.b200dp_mem_import(pfd, ctypes.byref(ph)))
                self.lib.b200dp_fd_close(pfd)
                handles[r] = ph.value
        self.lib.b200dp_fd_close(fd.value)
        ptrs = []
        for r in range(self.world):
            va = ctypes.c_uint64(0)
            self._ck(self.lib.b200dp_mem_map(self.dev_index, handles[r], padded, g,
                                             ctypes.byref(va)))
            ptrs.append(va.value)
        mc_ptr, mc_handle = 0, 0
        if use_mc:
            try:
                mc_ptr, mc_handle = self._setup_multicast(padded, g, handles[self.rank], mtag)
            except Exception as e:  # noqa: BLE001
                mc_ptr, mc_handle = 0, 0
                self._mc_fail = str(e)
            ok = [None] * self.world
            dist.all_gather_object(ok, mc_ptr != 0, group=self.group)
            if not all(ok):
                mc_ptr = 0
                self.multicast = False
        dist.barrier(group=self.group)
        buf = SymmBuffer(self, nbytes, padded, ptrs[self.rank], ptrs, mc_ptr,
                         {"mem": handles, "mc": mc_handle})
        self.buffers.append(buf)
        return buf

    def _setup_multicast(self, padded: int, align: int, my_handle: int, tag: int):
        mh = ctypes.c_uint64(0)
        if self.rank == 0:
            fd = ctypes.c_int(-1)
            self._ck(self.lib.b200dp_mc_create(self.world, padded, ctypes.byref(mh),
                                               ctypes.byref(fd)))
            for r in range(1, self.world):
                self._send_fd(r, fd.value, tag)
            self.lib.b200dp_fd_close(fd.value)
        else:
            pfd = self._recv_fd(0, tag)
            self._ck(self.lib.b200dp_mem_import(pfd, ctypes.byref(mh)))
            self.lib.b200dp_fd_close(pfd)
        self._ck(self.lib.b200dp_mc_add_device(mh.value, self.dev_index))
        dist.barrier(group=self.group)          # all devices added before any bind
        self._ck(self.lib.b200dp_mc_bind(mh.value, 0, my_handle, 0, padded))
        va = ctypes.c_uint64(0)
        self._ck(self.lib.b200dp_mem_map(self.dev_index, mh.value, padded, align, ctypes.byref(va)))
        return va.value, mh.value

    def alloc_tensor(self, numel: int, dtype: torch.dtype) -> torch.Tensor:
        es = torch.empty((), dtype=dtype).element_size()
        buf = self.alloc(numel * es)
        t = buf.tensor(dtype, numel)
        t._b200dp_symm = buf
        return t

    def find(self, t: torch.Tensor) -> Optional[Tuple[SymmBuffer, int]]:
        p, nb = t.data_ptr(), t.numel() * t.element_size()
        for b in self.buffers:
            if b.contains(p, nb):
                return b, p - b.local_ptr
        return None

    # ------------------------------------------------------------------ algorithm / grid choice
    def supports(self, dtype: torch.dtype) -> bool:
        return dtype in _DTYPE_CODE

    def pick_algo(self, nbytes: int, need_mc: bool = True) -> int:
        o = self.algo_override
        if o in ("oneshot", "one-shot", "0"):
            return ALGO_ONESHOT
        if o in ("twoshot", "two-shot", "1"):
            return ALGO_TWOSHOT
        if o in ("nvls", "2") and self.multicast and need_mc:
            return ALGO_NVLS
        # Table (runtime/tuning.py): one-shot only wins in the pure-latency regime; above it the
        # sliced kernels, and where the switch supports it the in-switch reduction (NVLS).
        from . import tuning
        return tuning.choose(self.world, nbytes, bool(self.multicast and need_mc))

    def pick_blocks(self, algo: int, nbytes: int) -> int:
        work = nbytes if algo == ALGO_ONESHOT else nbytes // max(self.world, 1)
        per_block = 512 * 16 * 2
        b = max(1, min((work + per_block - 1) // per_block, MAX_BLOCKS))
        cap = self.max_blocks or (32 if algo == ALGO_ONESHOT else (48 if algo == ALGO_NVLS else 64))
        return int(min(b, cap))

    # ------------------------------------------------------------------ launches
    def _lane(self, lane: int):
        """(staging buffer, signal channel) of a lane.  Lane 0 serves user collectives on the caller's
        stream; lane 1 is private to DistributedOptimizer's un-fused bucket path, which runs on its own
        side stream concurrently with user collectives — sharing one staging buffer and one set of
        barrier counters between two streams would corrupt both (ADVICE r1)."""
        if lane == 0:
            return self.stage, CH_USER
        if getattr(self, "stage_opt", None) is None:
            self.stage_opt = self.alloc(self.stage_bytes)      # collective: every rank takes this path together
        return self.stage_opt, CH_OPT

    def allreduce_(self, t: torch.Tensor, prescale: float = 1.0, postscale: float = 1.0,
                   algo: Optional[int] = None, lane: int = 0) -> torch.cuda.Event:
        """In-place sum-allreduce of ``t`` (scaled by prescale*postscale) on the current
        stream.  Zero-copy when ``t`` lives in symmetric memory; staged otherwise."""
        stream = torch.cuda.current_stream(self.device)
        stage, channel = self._lane(lane)
        scale = float(prescale) * float(postscale)
        es = t.element_size()
        work = t if t.is_contiguous() else t.contiguous()
        loc = self.find(work)
        vec = 16 // es
        if loc is not None and loc[1] % 16 == 0 and (work.numel() % vec == 0):
            buf, off = loc
            self._ar_symm(buf, off, work.numel(), work.dtype, scale, stream, algo, channel=channel)
        else:
            flat = work.view(-1)
            cap = (self.stage_bytes // es) // (vec * self.world) * (vec * self.world)
            st = stage.tensor(work.dtype)
            for lo in range(0, flat.numel(), cap):
                m = min(cap, flat.numel() - lo)
                mp = (m + vec - 1) // vec * vec
                st[:m].copy_(flat[lo:lo + m])
                if mp != m:
                    st[m:mp].zero_()
                self._ar_symm(stage, 0, mp, work.dtype, scale, stream, algo, user=True, channel=channel)
                flat[lo:lo + m].copy_(st[:m])
        if work is not t:
            t.copy_(work)
        ev = torch.cuda.Event()
        ev.record(stream)
        return ev

    def prepare_allreduce(self, t: torch.Tensor, scale: float = 1.0, algo: Optional[int] = None):
        """Pre-build the launch arguments for an in-place allreduce of a symmetric tensor and
        return a zero-argument callable that only does the ctypes launch on the current stream
        (host overhead ~2 us instead of ~12 us; used by benchmarks and tight loops)."""
        loc = self.find(t)
        es = t.element_size()
        assert loc is not None and loc[1] % 16 == 0 and t.numel() % (16 // es) == 0 and \
            t.is_contiguous(), "prepare_allreduce needs a 16B-aligned contiguous symmetric tensor"
        buf, off = loc
        nbytes = t.numel() * es
        a, algo = self._user_args(buf, off, t.numel(), nbytes, scale, algo, CH_USER)
        if algo == ALGO_ONESHOT:
            scratch = torch.empty(nbytes, dtype=torch.uint8, device=self.device)
            a.scratch, a.copy_back = scratch.data_ptr(), 1
        else:
            scratch = None
        blocks = self.pick_blocks(algo, nbytes)
        code = _DTYPE_CODE[t.dtype]
        fn, ctx_ref, a_ref = self.lib.b200dp_comm_allreduce, ctypes.byref(self.ctx), ctypes.byref(a)
        dev = self.device

        def launch(_keep=(a, scratch, t)):
            self._launched(fn(ctx_ref, a_ref, algo, code, blocks, 512, torch.cuda.current_stream(dev).cuda_stream))
        launch.algo = ALGO_NAMES[algo]
        launch.blocks = blocks
        return launch

    def _user_args(self, buf: SymmBuffer, off: int, numel: int, nbytes: int, scale: float, algo: Optional[int],
                   channel: int) -> Tuple[ARArgs, int]:
        """Argument block of an in-place sum-allreduce (no optimizer) of ``numel`` elements at byte ``off`` of
        ``buf``, and its algorithm: ``algo``, or the tuned choice; two-shot instead of NVLS where ``buf`` has no
        multicast address.  The caller supplies the one-shot scratch."""
        a = ARArgs()
        ptrs = buf.ptrs_at(off)
        for r in range(self.world):
            a.inp[r] = ptrs[r]
            a.out[r] = ptrs[r]
        a.n, a.scale, a.channel = numel, float(scale), channel
        a.h.kind = OPT_NONE
        algo = self.pick_algo(nbytes, need_mc=buf.mc_ptr != 0) if algo is None else algo
        if algo == ALGO_NVLS and buf.mc_ptr == 0:
            algo = ALGO_TWOSHOT
        if algo == ALGO_NVLS:
            a.in_mc = a.out_mc = buf.mc_ptr + off
        return a, algo

    def _ar_symm(self, buf: SymmBuffer, off: int, numel: int, dtype, scale, stream, algo,
                 user: bool = False, channel: int = CH_USER):
        nbytes = numel * torch.empty((), dtype=dtype).element_size()
        a, algo = self._user_args(buf, off, numel, nbytes, scale, algo, channel)
        if algo == ALGO_ONESHOT:
            key = "scratch" if channel == CH_USER else "scratch_opt"
            sc = getattr(self, key, None)
            if sc is None or nbytes > sc.numel():
                sc = torch.empty(max(nbytes, 1 << 20), dtype=torch.uint8, device=self.device)
                setattr(self, key, sc)
            a.scratch = sc.data_ptr()
            a.copy_back = 1
        self.launch_allreduce(a, algo, dtype, nbytes, stream)

    # ------------------------------------------------------------------ reduce-scatter / all-gather / all-to-all
    def _coll(self, mode: int, a: CollArgs, dtype, work_bytes: int, stream):
        blocks = self._coll_blocks(work_bytes)
        self._launched(self.lib.b200dp_comm_collective(ctypes.byref(self.ctx), ctypes.byref(a), mode,
                                                       _DTYPE_CODE.get(dtype, 0), blocks, 512, stream.cuda_stream))

    def _coll_blocks(self, work_bytes: int) -> int:
        return max(1, min((work_bytes + 512 * 16 * 2 - 1) // (512 * 16 * 2), self.max_blocks or 48))

    def _group(self, members) -> Tuple[List[int], int]:
        """(members as a list, this rank's index in it); the C entry point checks the rest of the list."""
        members = [int(w) for w in members]
        if self.rank not in members:
            raise ValueError(f"rank {self.rank} is not a member of the group {members}")
        return members, members.index(self.rank)

    def _group_coll(self, mode: int, a: GroupCollArgs, dtype, work_bytes: int, stream):
        self._launched(self.lib.b200dp_comm_group_collective(ctypes.byref(self.ctx), ctypes.byref(a), mode,
                                                             _DTYPE_CODE.get(dtype, 0), self._coll_blocks(work_bytes),
                                                             512, stream.cuda_stream))

    def reducescatter(self, src: torch.Tensor, out: torch.Tensor, scale: float = 1.0,
                      members=None) -> torch.cuda.Event:
        """``out`` (numel = src.numel() / world) = scale * sum over ranks of chunk ``rank`` of ``src``.
        ``src`` is staged into symmetric memory (chunk-major slabs when larger than the staging
        buffer); each rank then reads ONLY its own chunk from every peer (or lets the switch sum it).
        ``members`` (world ranks, ascending): the same among those ranks only, with the group's size and this
        rank's index in it in place of the world's; never multicast."""
        stream = torch.cuda.current_stream(self.device)
        if members is not None:
            members, gi = self._group(members)
        W, es = (self.world if members is None else len(members)), src.element_size()
        vec = 16 // es
        chunk = src.numel() // W
        assert src.numel() == chunk * W and out.numel() == chunk and chunk % vec == 0
        s2, o1 = src.reshape(W, chunk), out.reshape(chunk)
        cap = (self.stage_bytes // es) // (W * vec) * vec            # elements per rank chunk per slab
        st = self.stage.tensor(src.dtype)
        for lo in range(0, chunk, cap):
            m = min(cap, chunk - lo)
            st[: W * m].view(W, m).copy_(s2[:, lo:lo + m])
            dst = o1[lo:lo + m]
            if members is not None:
                a = group_coll_args(members, gi, [self.stage.peer_ptrs[w] for w in members],
                                    [dst.data_ptr() if g == gi else 0 for g in range(W)], m, scale)
                self._group_coll(COLL_REDUCE_SCATTER, a, src.dtype, m * es, stream)
                continue
            a = CollArgs()
            for r in range(W):
                a.src[r] = self.stage.peer_ptrs[r]
            a.dst[self.rank] = dst.data_ptr()
            a.chunk, a.scale, a.channel = m, float(scale), CH_USER
            a.use_mc = 1 if (self.stage.mc_ptr and m * es >= (64 << 10)) else 0
            a.src_mc = self.stage.mc_ptr
            self._coll(COLL_REDUCE_SCATTER, a, src.dtype, m * es, stream)
        ev = torch.cuda.Event()
        ev.record(stream)
        return ev

    def allgather(self, src: torch.Tensor, out: torch.Tensor, members=None) -> torch.cuda.Event:
        """``out`` (world * src.numel()) = concatenation of every rank's ``src`` (equal sizes, 16-byte
        multiple).  Each rank pushes its chunk into slot ``rank`` of every peer's staging buffer.
        ``members`` (world ranks, ascending): the concatenation over those ranks only, in group-rank order;
        never multicast."""
        return self._push(COLL_ALLGATHER, src, out, members)

    def alltoall(self, src: torch.Tensor, out: torch.Tensor) -> torch.cuda.Event:
        """Equal-split all-to-all: chunk j of ``src`` lands in slot ``rank`` of rank j's ``out``."""
        return self._push(COLL_ALLTOALL, src, out)

    def _push(self, mode: int, src: torch.Tensor, out: torch.Tensor, members=None) -> torch.cuda.Event:
        stream = torch.cuda.current_stream(self.device)
        if members is not None:
            members, gi = self._group(members)
        W = self.world if members is None else len(members)
        sb = src.reshape(-1).view(torch.uint8)
        ob = out.reshape(-1).view(torch.uint8)
        chunk = sb.numel() if mode == COLL_ALLGATHER else sb.numel() // W     # bytes per (src, dst) pair
        assert chunk % 16 == 0 and ob.numel() == chunk * W
        cap = (self.stage_bytes // W) // 16 * 16
        st = self.stage.tensor(torch.uint8)
        o2 = ob.view(W, chunk)
        for lo in range(0, chunk, cap):
            m = min(cap, chunk - lo)
            if mode == COLL_ALLGATHER:
                piece = sb[lo:lo + m]
            else:                                   # pack the W sub-chunks of this slab contiguously
                piece = sb.view(W, chunk)[:, lo:lo + m].contiguous().view(-1)
            if members is None:
                a = CollArgs()
                a.src[self.rank] = piece.data_ptr()
                for r in range(W):
                    a.dst[r] = self.stage.peer_ptrs[r]
                a.chunk, a.channel = m // 16, CH_USER
                a.use_mc = 1 if (mode == COLL_ALLGATHER and self.stage.mc_ptr and m >= (64 << 10)) else 0
                a.dst_mc = self.stage.mc_ptr
                self._coll(mode, a, torch.uint8, m, stream)
            else:
                a = group_coll_args(members, gi, [piece.data_ptr() if g == gi else 0 for g in range(W)],
                                    [self.stage.peer_ptrs[w] for w in members], m // 16)
                self._group_coll(mode, a, torch.uint8, m, stream)
            o2[:, lo:lo + m].copy_(st[: W * m].view(W, m))
            piece.record_stream(stream) if piece.data_ptr() != sb.data_ptr() else None
        ev = torch.cuda.Event()
        ev.record(stream)
        return ev

    def broadcast_(self, t: torch.Tensor, root: int) -> torch.cuda.Event:
        stream = torch.cuda.current_stream(self.device)
        loc = self.find(t)
        nbytes = t.numel() * t.element_size()
        if loc is not None and loc[1] % 16 == 0 and nbytes % 16 == 0:
            self._bcast(loc[0], loc[1], nbytes, root, stream)
        else:
            flat = t.view(-1).view(torch.uint8) if t.is_contiguous() else None
            if flat is None:
                raise RuntimeError("broadcast_ needs a contiguous tensor")
            st = self.stage.tensor(torch.uint8)
            cap = self.stage_bytes
            for lo in range(0, nbytes, cap):
                m = min(cap, nbytes - lo)
                mp = (m + 15) // 16 * 16
                if self.rank == root:
                    st[:m].copy_(flat[lo:lo + m])
                self._bcast(self.stage, 0, mp, root, stream)
                if self.rank != root:
                    flat[lo:lo + m].copy_(st[:m])
        ev = torch.cuda.Event()
        ev.record(stream)
        return ev

    def _bcast(self, buf: SymmBuffer, off: int, nbytes: int, root: int, stream):
        a = BcastArgs()
        ptrs = buf.ptrs_at(off)
        for r in range(self.world):
            a.buf[r] = ptrs[r]
        a.buf_mc = buf.mc_ptr + off if buf.mc_ptr else 0
        a.nbytes, a.root, a.channel = nbytes, root, CH_BCAST
        a.use_mc = 1 if (buf.mc_ptr and os.environ.get("B200DP_BCAST_P2P", "0") != "1") else 0
        blocks = max(1, min((nbytes + 512 * 16 * 4 - 1) // (512 * 16 * 4), 32))
        self._launched(self.lib.b200dp_comm_broadcast(ctypes.byref(self.ctx), ctypes.byref(a), blocks, 512,
                                                      stream.cuda_stream))

    # ------------------------------------------------------------------ watchdog / teardown
    def check_errors(self):
        """Raise if a kernel's bounded spin-wait expired (a peer died or diverged)."""
        if self._mailbox[0] != 0:
            peer, block, ch = self._mailbox[1], self._mailbox[2], self._mailbox[3]
            from ..torch.mpi_ops import HorovodInternalError
            raise HorovodInternalError(
                f"collective watchdog: rank {self.rank} timed out waiting for rank {peer} "
                f"(block {block}, channel {ch}) — a peer died, hung or ran a different "
                f"collective sequence")

    def reset_errors(self):
        """Collective: clear the watchdog mailbox and restart the cross-rank barrier protocol from zero
        (signal pads + epoch counters), so a retry after a failed collective (``hvd.elastic.run``) does
        not trip over the stale state of the run that timed out."""
        torch.cuda.synchronize(self.device)
        dist.barrier(group=self.group)
        for i in range(4):
            self._mailbox[i] = 0
        self.sig.tensor(torch.int32).zero_()
        self.epoch.zero_()
        torch.cuda.synchronize(self.device)
        dist.barrier(group=self.group)

    def close(self):
        """Release everything this runtime mapped: multicast bindings, peer mappings and the cuMem
        handles of every symmetric allocation (``hvd.shutdown(); hvd.init()`` cycles — what
        ``hvd.elastic.run`` does after a failure — must not leak 64 MiB of staging plus all arenas).
        Tensors that still alias a released range must not be used afterwards; the fused engine drops
        its arena views in ``FusedEngine.release()``, which ``hvd.shutdown()`` calls first."""
        try:
            torch.cuda.synchronize(self.device)
        except Exception:
            pass
        for buf in list(getattr(self, "buffers", [])):
            try:
                self.free(buf)
            except Exception:      # noqa: BLE001 - best effort at teardown
                pass
        self.buffers = []
        self.stage = self.stage_opt = None
        if getattr(self, "_sock", -1) >= 0:
            self.lib.b200dp_fd_close(self._sock)
            self._sock = -1

    def free(self, buf: SymmBuffer):
        """Unmap and release one symmetric allocation (local mapping, every peer mapping, the multicast
        mapping and binding).  Local operation; call it on every rank."""
        if buf._handles is None:
            return
        buf._bytes = None
        mc = buf._handles.get("mc", 0)
        if buf.mc_ptr:
            self.lib.b200dp_mem_unmap(buf.mc_ptr, buf.padded)
            if mc:
                self.lib.b200dp_mc_unbind(mc, self.dev_index, 0, buf.padded)
        if mc:
            self.lib.b200dp_mem_release(mc)
        for r, va in enumerate(buf.peer_ptrs):
            self.lib.b200dp_mem_unmap(va, buf.padded)
        for r, h in buf._handles.get("mem", {}).items():
            self.lib.b200dp_mem_release(h)
        buf._handles = None
        buf.mc_ptr = 0
        buf.peer_ptrs = []
        if buf in self.buffers:
            self.buffers.remove(buf)
