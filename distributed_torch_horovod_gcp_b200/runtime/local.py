"""World-size-1 flavour of the symmetric runtime: same kernels (``ctx.world == 1`` skips the
cross-rank barriers), plain device memory instead of cuMem-shared allocations.  Lets the
fused scale+optimizer epilogue (K7) run as a single flat multi-tensor update on one GPU
(``B200DP_FUSED_SINGLE=1``) and keeps one code path for 1..8 GPUs."""
from __future__ import annotations

import ctypes
import os
from typing import List, Optional

import torch

from . import lib as _lib
from . import symm as S


class _LocalBuffer:
    def __init__(self, rt, nbytes: int):
        self.rt, self.nbytes, self.padded = rt, nbytes, (nbytes + 255) // 256 * 256
        self._bytes = torch.zeros(self.padded, dtype=torch.uint8, device=rt.device)
        self.local_ptr = self._bytes.data_ptr()
        self.peer_ptrs = [self.local_ptr]
        self.mc_ptr = 0

    def tensor(self, dtype, numel=None, byte_offset=0):
        es = torch.empty((), dtype=dtype).element_size()
        if numel is None:
            numel = (self.nbytes - byte_offset) // es
        return self._bytes[byte_offset: byte_offset + numel * es].view(dtype)

    def contains(self, ptr, nbytes):
        return self.local_ptr <= ptr and ptr + nbytes <= self.local_ptr + self.padded

    def ptrs_at(self, off):
        return [self.local_ptr + off]


class LocalRuntime(S.KernelLauncher):
    _inst: Optional["LocalRuntime"] = None

    @classmethod
    def get(cls) -> Optional["LocalRuntime"]:
        if cls._inst is not None:
            return cls._inst
        if not torch.cuda.is_available():
            return None
        lib = _lib.load_comm()
        if lib is None:
            return None
        self = object.__new__(cls)
        self.lib = lib
        S.SymmRuntime._bind(self)
        self.rank, self.world, self.multicast = 0, 1, False
        self.device = torch.device("cuda", torch.cuda.current_device())
        self.epoch = torch.zeros(S.NUM_CHANNELS * S.MAX_BLOCKS * S.MAX_RANKS, dtype=torch.int32,
                                 device=self.device)
        hp, dp = ctypes.c_uint64(0), ctypes.c_uint64(0)
        if lib.b200dp_host_mailbox(64, ctypes.byref(hp), ctypes.byref(dp)) != 0:
            return None
        self._mailbox = (ctypes.c_int * 16).from_address(hp.value)
        self.ctx = S.CommCtx()
        self._sig = torch.zeros(S.NUM_CHANNELS * S.MAX_BLOCKS * S.MAX_RANKS, dtype=torch.int32,
                                device=self.device)
        self.ctx.sig[0] = self._sig.data_ptr()
        self.ctx.epoch, self.ctx.err = self.epoch.data_ptr(), dp.value
        self.ctx.timeout_ns, self.ctx.rank, self.ctx.world = int(20e9), 0, 1
        self.max_blocks = int(os.environ.get("B200DP_COMM_BLOCKS", "0"))
        self.algo_override = "oneshot"
        self.buffers: List[_LocalBuffer] = []
        self.launches = 0
        cls._inst = self
        return self

    def alloc(self, nbytes: int, multicast: bool = True) -> _LocalBuffer:
        b = _LocalBuffer(self, nbytes)
        self.buffers.append(b)
        return b

    def pick_algo(self, nbytes: int, need_mc: bool = True) -> int:
        return S.ALGO_ONESHOT

    def pick_blocks(self, algo: int, nbytes: int) -> int:
        per_block = 512 * 16 * 4
        return int(max(1, min((nbytes + per_block - 1) // per_block, self.max_blocks or 128)))

    def allreduce_(self, t, prescale=1.0, postscale=1.0, algo=None):
        if prescale * postscale != 1.0:
            t.mul_(prescale * postscale)
        ev = torch.cuda.Event()
        ev.record(torch.cuda.current_stream(self.device))
        return ev

    def check_errors(self):
        return

    def close(self):
        return
