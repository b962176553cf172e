"""Minimal elastic-state API (Horovod ``hvd.elastic`` shape): in-memory commit / restore /
sync of model + optimizer, and a ``run`` decorator that rolls back to the last commit when
a collective fails (``HorovodInternalError``).

The reference enables none of this (SURVEY.md §5.3); it is provided for surface parity and
as the failure-recovery hook for the kernel watchdog (a bounded spin-wait in the sm_90a
kernels sets an error flag -> ``HorovodInternalError``).

Resizing is restart-based (launch/run.py elastic mode): ``state.check_host_updates()`` lets rank 0
re-run the launcher's host-discovery script; when the host set differs from the one the job was
launched on every rank raises ``HostsUpdatedInterrupt``, ``run`` persists the last commit
(``B200DP_ELASTIC_STATE_DIR``) and the workers exit with code 75, which makes the launcher relaunch
on the new host set; the new workers start from the persisted commit.
"""
from __future__ import annotations

import copy
import functools

import torch

from .mpi_ops import HorovodInternalError

RESTART_EXIT = 75


class HostsUpdatedInterrupt(RuntimeError):
    """The set of available hosts changed (Horovod's exception of the same name)."""

    def __init__(self, skip_sync: bool = False):
        super().__init__("hosts updated")
        self.skip_sync = skip_sync


class State:
    def __init__(self, **kwargs):
        self._attrs = dict(kwargs)
        for k, v in kwargs.items():
            setattr(self, k, v)
        self._saved = {}
        self._reset_callbacks = []
        self.save()

    def register_reset_callbacks(self, callbacks):
        self._reset_callbacks.extend(callbacks)

    def on_reset(self):
        for cb in self._reset_callbacks:
            cb()

    def save(self):
        self._saved = {k: copy.deepcopy(getattr(self, k)) for k in self._attrs}

    def restore(self):
        for k, v in self._saved.items():
            setattr(self, k, copy.deepcopy(v))

    def commit(self):
        self.save()

    def check_host_updates(self):
        """Raise ``HostsUpdatedInterrupt`` on every rank when the launcher's discovery script reports a
        host set different from the one this job runs on.  No-op outside elastic launches; rank 0 runs
        the script at most every ``B200DP_DISCOVERY_INTERVAL_S`` seconds (default 5)."""
        import os
        import subprocess
        import time
        script = os.environ.get("B200DP_DISCOVERY_SCRIPT")
        if not script:
            return None
        from .. import _state
        from .functions import broadcast_object
        changed = False
        if _state.rank() == 0:
            now = time.time()
            every = float(os.environ.get("B200DP_DISCOVERY_INTERVAL_S", "5"))
            if now - getattr(self, "_last_discovery", 0.0) >= every:
                self._last_discovery = now
                try:
                    from ..launch.run import discover_hosts
                    spec = ",".join(f"{h}:{s}" for h, s in discover_hosts(script))
                    changed = spec != os.environ.get("B200DP_ELASTIC_HOSTS", spec)
                except (RuntimeError, subprocess.SubprocessError, OSError):
                    changed = False
        changed = broadcast_object(changed, 0)
        if changed:
            raise HostsUpdatedInterrupt()
        return None

    # -- persistence across an elastic relaunch ------------------------------------------
    def _persist_path(self):
        import os
        d = os.environ.get("B200DP_ELASTIC_STATE_DIR")
        return os.path.join(d, "state.pt") if d else None

    def persist(self):
        """Rank 0 writes the last commit to disk (atomic rename)."""
        import os
        from .. import _state
        path = self._persist_path()
        if path is None or _state.rank() != 0:
            return
        tmp = path + ".tmp"
        torch.save(self._persist_payload(), tmp)
        os.replace(tmp, path)

    def load_persisted(self) -> bool:
        import os
        path = self._persist_path()
        if path is None or not os.path.exists(path):
            return False
        self._load_payload(torch.load(path, map_location="cpu", weights_only=False))
        return True

    def _persist_payload(self):
        return {"attrs": dict(self._saved)}

    def _load_payload(self, payload):
        self._saved = dict(payload["attrs"])
        self.restore()

    def sync(self):
        from .functions import broadcast_object
        for k in self._attrs:
            setattr(self, k, broadcast_object(getattr(self, k), 0))


class TorchState(State):
    """State of a model + optimizer (+ arbitrary picklable kwargs such as epoch/batch)."""

    def __init__(self, model=None, optimizer=None, **kwargs):
        self.model, self.optimizer = model, optimizer
        self._model_sd, self._opt_sd = None, None
        super().__init__(**kwargs)

    def save(self):
        super().save()
        if self.model is not None:
            self._model_sd = {k: v.detach().clone() for k, v in self.model.state_dict().items()}
        if self.optimizer is not None:
            eng = getattr(self.optimizer, "fused_engine", None)
            if eng is not None:
                eng.export_state()
            self._opt_sd = copy.deepcopy(self.optimizer.state_dict())

    def restore(self):
        super().restore()
        if self.model is not None and self._model_sd is not None:
            with torch.no_grad():
                for k, v in self.model.state_dict().items():
                    v.copy_(self._model_sd[k])
        if self.optimizer is not None and self._opt_sd is not None:
            self.optimizer.load_state_dict(copy.deepcopy(self._opt_sd))
            eng = getattr(self.optimizer, "fused_engine", None)
            if eng is not None:
                eng.params_changed()
                eng.import_state()

    def _persist_payload(self):
        return {"attrs": dict(self._saved), "model": self._model_sd, "opt": self._opt_sd}

    def _load_payload(self, payload):
        dev = next(self.model.parameters()).device if self.model is not None else None
        if payload.get("model") is not None and dev is not None:
            self._model_sd = {k: v.to(dev) for k, v in payload["model"].items()}
        self._opt_sd = payload.get("opt")
        self._saved = dict(payload["attrs"])
        self.restore()

    def sync(self):
        from .functions import broadcast_parameters, broadcast_optimizer_state
        if self.model is not None:
            broadcast_parameters(self.model.state_dict(), root_rank=0)
        if self.optimizer is not None:
            broadcast_optimizer_state(self.optimizer, root_rank=0)
        super().sync()


class ObjectState(State):
    """State of arbitrary picklable python objects (Horovod ``hvd.elastic.ObjectState``)."""


class ElasticSampler(torch.utils.data.Sampler):
    """Sharded sampler that remembers which indices were already processed in the current epoch,
    so that after a reset (rollback / world-size change) the remaining samples are re-partitioned
    over the new set of ranks (Horovod ``hvd.elastic.ElasticSampler`` shape)."""

    def __init__(self, dataset, shuffle: bool = True, seed: int = 0):
        self.dataset, self.shuffle, self.seed = dataset, shuffle, seed
        self.epoch = 0
        self.processed_indices = set()
        self.reset()

    def set_epoch(self, epoch: int):
        self.epoch = epoch
        self.processed_indices = set()
        self.reset()

    def record_batch(self, batch_idx: int, batch_size: int):
        lo = batch_idx * batch_size
        self.processed_indices.update(self.indices[lo: lo + batch_size])

    def load_state_dict(self, sd):
        self.epoch = sd["epoch"]
        self.processed_indices = set(sd["processed_indices"])
        self.reset()

    def state_dict(self):
        return {"epoch": self.epoch, "processed_indices": sorted(self.processed_indices)}

    def reset(self):
        from .. import _state
        self.num_replicas = _state.size() if _state.is_initialized() else 1
        self.rank = _state.rank() if _state.is_initialized() else 0
        remaining = [i for i in range(len(self.dataset)) if i not in self.processed_indices]
        if self.shuffle:
            g = torch.Generator().manual_seed(self.seed + self.epoch)
            perm = torch.randperm(len(remaining), generator=g).tolist()
            remaining = [remaining[i] for i in perm]
        self.num_samples = -(-len(remaining) // self.num_replicas) if remaining else 0
        total = self.num_samples * self.num_replicas
        remaining += remaining[: total - len(remaining)]
        self.indices = remaining[self.rank: total: self.num_replicas]

    def __iter__(self):
        return iter(self.indices)

    def __len__(self):
        return len(self.indices)


def run(func):
    """Decorator: ``func(state, *args)`` is retried from the last commit after a collective
    failure.  ``B200DP_ELASTIC_MAX_RETRIES`` bounds the retries (default 3)."""
    import os

    @functools.wraps(func)
    def wrapper(state, *args, **kwargs):
        import sys
        retries = int(os.environ.get("B200DP_ELASTIC_MAX_RETRIES", "3"))
        from .. import _state
        if _state.rank() == 0:
            state.load_persisted()          # resuming after an elastic relaunch
        state.sync()
        while True:
            try:
                return func(state, *args, **kwargs)
            except HostsUpdatedInterrupt:
                # the world is about to change: keep the last commit, hand control back to the launcher
                state.persist()
                from . import mpi_ops
                try:
                    mpi_ops.barrier()
                except Exception:      # noqa: BLE001
                    pass
                sys.stdout.flush()
                sys.stderr.flush()
                os._exit(RESTART_EXIT)
            except HorovodInternalError:
                if retries <= 0:
                    raise
                retries -= 1
                symm = _state.runtime().symm
                if symm is not None:
                    symm.reset_errors()     # clear the watchdog mailbox and the barrier counters (collective)
                state.restore()
                state.on_reset()
                state.sync()
    return wrapper
