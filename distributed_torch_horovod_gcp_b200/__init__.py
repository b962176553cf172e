"""distributed_torch_horovod_gcp_b200 — an H100-native data-parallel training framework.

A from-scratch replacement for the slice of Horovod that the reference
``app/torch_train.py`` exercises (reference: app/torch_train.py:17,210-266), designed
for multi-GPU H100 nodes over NVLink / NVSwitch:

* ``distributed_torch_horovod_gcp_b200.torch`` — the ``hvd``-shaped public API
  (``init/rank/size/local_rank/DistributedOptimizer/broadcast_parameters/allreduce``…)
* ``.runtime``   — C++ symmetric-memory runtime (cuMem VMM + multicast, fd exchange)
* ``.ops``       — hand-written sm_90a kernels (fused allreduce+optimizer, wgmma GEMM,
  implicit-GEMM convolution, flash attention, persistent LSTM recurrence, batch-norm / layer-norm /
  pooling) and their autograd wrappers
* ``.parallel``  — bucket planner, backward hooks, side-stream overlap
* ``.models``    — LSTM (reference model), ResNet-18/50/152, ViT-B/16
* ``.launch``    — ``horovodrun``-shaped launcher (``-np N -H host:slots``)

Usage mirrors Horovod::

    import distributed_torch_horovod_gcp_b200.torch as hvd
    hvd.init()
"""

__version__ = "0.2.0"

from . import _state  # noqa: F401  (process-wide runtime state)
