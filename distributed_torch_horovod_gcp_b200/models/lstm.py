"""LSTM regressor — the reference model (app/torch_train.py:107-206; SURVEY.md §2.1 C6).

Architecture (parity): ``nn.LSTM(n_features -> h_size, n_layers, bidirectional?,
batch_first, dropout)`` -> ``Linear(h*dirs -> h)`` -> ``Linear(h -> 64)`` -> ``Linear(64 -> 1)`` with
NO activations between the linears (app/torch_train.py:199-205); fresh random ``(h0, c0)``
every forward (app/torch_train.py:179-193); the last timestep is selected
(app/torch_train.py:196); output shape ``[B, 1, 1]``.  ``state_dict`` keys are identical to
the reference's (``lstm.weight_ih_l0`` … ``linear3.bias``) so ``broadcast_parameters``
moves the same 10 tensors / 1 480 196 bytes.

H100-first changes (SURVEY.md §2.6 S2/S4, §7.3):
  * ``(h0, c0)`` come from the device generator (no CPU randn + pageable H2D + sync per
    step), the last-step gather is a slice (no host-built index tensor);
  * the recurrence and the head are ``ops.functional.lstm`` and ``ops.functional.lstm_head``, each of
    which chooses its kernel.  On an sm_90 device (fp32, hidden size 256, any number of layers, one or two
    directions, 1..512 input features, inter-layer dropout in [0, 1]) forward/backward run on the persistent
    cluster LSTM kernels (K5: ``ops/lstm_rec.py``, csrc/lstm_rec_sm90.cu — tf32 wgmma, W_hh resident in shared
    memory, h exchanged through DSMEM; the two directions of a layer run as separate clusters of one launch)
    and, for batches up to 1024, the chained-GEMM head (K6: ``ops/lstm_fused.py``; larger batches use torch's
    linears).  Other hidden sizes, wider inputs and non-fp32 weights use cuDNN / cuBLAS, which is also the
    numerics oracle; ``fused=False`` takes cuDNN / cuBLAS for every shape.
"""
from __future__ import annotations

import warnings
from typing import Callable, Optional, Sequence

import torch
from torch import nn

from ..ops import functional as F2


class LSTM(nn.Module):
    """implements an lstm - a single/multilayer uni/bi directional lstm"""

    def __init__(self, n_features, window_size, output_size, h_size, n_layers=1,
                 bidirectional=False, device=torch.device('cpu'),
                 initializers: Optional[Sequence[Callable]] = None, fused: Optional[bool] = None,
                 dropout: float = 0.0):
        super().__init__()
        self.n_features = n_features
        self.window_size = window_size
        self.output_size = output_size
        self.h_size = h_size
        self.n_layers = n_layers
        self.directions = 2 if bidirectional else 1
        self.device = torch.device(device)

        self.lstm = nn.LSTM(input_size=n_features, hidden_size=h_size, num_layers=n_layers,
                            bidirectional=bidirectional, batch_first=True, dropout=dropout)
        self.hidden = None
        self.linear = nn.Linear(self.h_size * self.directions, self.h_size)
        self.linear2 = nn.Linear(self.h_size, 64)
        self.linear3 = nn.Linear(64, output_size)

        self.layers = [self.lstm, self.linear, self.linear2, self.linear3]
        self.initializers = list(initializers) if initializers else []
        self._initialize_all_layers()
        self._fused = fused

    # -- initializer plumbing (reference C6a: a stub there; functional here) ---------------
    def _initialize_all_layers(self):
        """One initializer -> used for all layers (with a warning); one per layer -> applied
        pairwise; any other count -> error; none -> default init.  Layers are moved to
        ``self.device`` in every case (app/torch_train.py:139-167)."""
        n_init, n_layers = len(self.initializers), len(self.layers)
        if n_init == 1 and n_layers != 1:
            warnings.warn("only one initializer: {} was provided for {} layers, the initializer "
                          "will be used for all layers".format(self.initializers[0], n_layers))
            for layer in self.layers:
                self._initialize_layer(self.initializers[0], layer)
        elif n_init == n_layers:
            for init, layer in zip(self.initializers, self.layers):
                self._initialize_layer(init, layer)
        elif n_init != 0:
            raise Exception("{} initializers were provided for {} layers, need to provide an "
                            "initializer for each layer".format(n_init, n_layers))
        else:
            for layer in self.layers:
                self._initialize_layer(None, layer)

    def _initialize_layer(self, initializer, layer):
        if initializer:
            with torch.no_grad():
                for p in layer.parameters():
                    if p.dim() >= 2:
                        initializer(p)
        layer.to(self.device)

    def _make_tensor(self, tensor_type, *args, **kwargs):
        """returns a tensor of ``tensor_type`` ('long' | 'float') on the model's device."""
        dtype = {"float": torch.float32, "long": torch.int64}[tensor_type]
        return torch.tensor(*args, dtype=dtype, device=self.device, **kwargs)

    def init_hidden(self, batch_size):
        dev = self.lstm.weight_hh_l0.device
        dt = self.lstm.weight_hh_l0.dtype
        shape = (self.n_layers * self.directions, batch_size, self.h_size)
        return (torch.randn(shape, device=dev, dtype=dt), torch.randn(shape, device=dev, dtype=dt))

    def forward(self, input):
        self.hidden = self.init_hidden(input.size(0))
        if self._fused is False:
            lstm, head = F2.lstm_reference, F2.lstm_head_reference
        else:
            lstm, head = F2.lstm, F2.lstm_head
        lstm_output, self.hidden = lstm(input, self.lstm, self.hidden)
        return head(lstm_output, self.window_size - 1, self.linear, self.linear2, self.linear3)
