"""Synthetic input pipelines for the [DRIVER] benchmark configs (BASELINE.json: "synthetic
data of the benchmark's shape").

``SyntheticImageBatches`` keeps a small ring of *pinned host* batches and stages them to the
device on a copy stream (double-buffered), so an end-to-end step really contains the H2D
copy of that step's inputs — the e2e number in bench.py counts these bytes.

``SyntheticTokenBatches`` draws language-model token batches directly on the device.

``DeviceBatchLoader`` is the H100-first replacement for the reference's
DataLoader+DistributedSampler on tiny tensors (app/torch_train.py:248-251): the whole
(small) training set lives on the device, the sharded permutation is computed once per
epoch, and batches are gathered on-device — no worker processes, no per-batch H2D.
"""
from __future__ import annotations

import math
from typing import Iterator, Optional, Tuple

import torch


class SyntheticImageBatches:
    def __init__(self, batch: int, shape=(3, 224, 224), num_classes: int = 1000,
                 device: Optional[torch.device] = None, dtype=torch.bfloat16, ring: int = 4,
                 channels_last: bool = True, seed: int = 0):
        self.batch, self.shape, self.device, self.dtype = batch, shape, device, dtype
        g = torch.Generator().manual_seed(seed)
        pin = device is not None and device.type == "cuda"
        self.host_x, self.host_y = [], []
        for _ in range(ring):
            x = torch.randn((batch,) + tuple(shape), generator=g).to(dtype)
            if channels_last:
                x = x.contiguous(memory_format=torch.channels_last)
            y = torch.randint(0, num_classes, (batch,), generator=g)
            if pin:
                x, y = x.pin_memory(), y.pin_memory()
            self.host_x.append(x)
            self.host_y.append(y)
        self.copy_stream = torch.cuda.Stream() if pin else None
        self._i = 0
        self._staged = None
        self.bytes_per_batch = self.host_x[0].numel() * self.host_x[0].element_size() + \
            self.host_y[0].numel() * self.host_y[0].element_size()

    def _stage(self):
        k = self._i % len(self.host_x)
        self._i += 1
        if self.copy_stream is None:
            return self.host_x[k], self.host_y[k], None
        with torch.cuda.stream(self.copy_stream):
            x = self.host_x[k].to(self.device, non_blocking=True)
            y = self.host_y[k].to(self.device, non_blocking=True)
            ev = torch.cuda.Event()
            ev.record(self.copy_stream)
        return x, y, ev

    def next(self) -> Tuple[torch.Tensor, torch.Tensor]:
        """Return the staged batch (waiting on its copy) and start staging the next one."""
        if self._staged is None:
            self._staged = self._stage()
        x, y, ev = self._staged
        if ev is not None:
            torch.cuda.current_stream().wait_event(ev)
            x.record_stream(torch.cuda.current_stream())
            y.record_stream(torch.cuda.current_stream())
        self._staged = self._stage()
        return x, y


class SyntheticTokenBatches:
    """Language-model batches of uniform random tokens drawn on ``device`` from a seeded generator:
    ``next()`` returns (inputs [B, S], targets [B * S]), both int64, the targets being the inputs
    shifted left by one position (drawn as one [B, S + 1] sequence)."""

    def __init__(self, batch: int, seq_len: int, vocab: int, device=None, seed: int = 0):
        self.batch, self.seq_len, self.vocab = batch, seq_len, vocab
        self.device = torch.device(device) if device is not None else torch.device("cpu")
        self.gen = torch.Generator(device=self.device).manual_seed(seed)

    def next(self) -> Tuple[torch.Tensor, torch.Tensor]:
        t = torch.randint(0, self.vocab, (self.batch, self.seq_len + 1), generator=self.gen,
                          device=self.device, dtype=torch.int64)
        return t[:, :-1], t[:, 1:].reshape(-1)


class DeviceBatchLoader:
    """Device-resident sharded mini-batch iterator with DistributedSampler semantics
    (pads to a multiple of ``num_replicas``; strided shard; ``shuffle=True, seed=0`` and
    — reference parity — the SAME permutation every epoch unless ``set_epoch`` is called)."""

    def __init__(self, X: torch.Tensor, Y: torch.Tensor, batch_size: int, num_replicas: int = 1,
                 rank: int = 0, shuffle: bool = True, seed: int = 0, drop_last: bool = False,
                 device: Optional[torch.device] = None):
        self.device = device or X.device
        self.X = X.to(self.device, non_blocking=True)
        self.Y = Y.to(self.device, non_blocking=True)
        self.batch_size, self.num_replicas, self.rank = batch_size, num_replicas, rank
        self.shuffle, self.seed, self.epoch, self.drop_last = shuffle, seed, 0, drop_last
        n = len(X)
        self.num_samples = math.ceil(n / num_replicas)
        self.total_size = self.num_samples * num_replicas

    def set_epoch(self, epoch: int):
        self.epoch = epoch

    def _indices(self) -> torch.Tensor:
        n = len(self.X)
        if self.shuffle:
            g = torch.Generator().manual_seed(self.seed + self.epoch)
            idx = torch.randperm(n, generator=g)
        else:
            idx = torch.arange(n)
        pad = self.total_size - n
        if pad > 0:
            reps = math.ceil(pad / max(n, 1))
            idx = torch.cat([idx, idx.repeat(reps)[:pad]])
        return idx[self.rank:self.total_size:self.num_replicas]

    def __len__(self):
        if self.drop_last:
            return self.num_samples // self.batch_size
        return math.ceil(self.num_samples / self.batch_size)

    def __iter__(self) -> Iterator[Tuple[torch.Tensor, torch.Tensor]]:
        idx = self._indices().to(self.device, non_blocking=True)
        for b in range(len(self)):
            sel = idx[b * self.batch_size:(b + 1) * self.batch_size]
            yield self.X.index_select(0, sel), self.Y.index_select(0, sel)
