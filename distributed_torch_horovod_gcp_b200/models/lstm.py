"""LSTM regressor — the reference model (app/torch_train.py:107-206; SURVEY.md §2.1 C6).

Architecture (parity): ``nn.LSTM(n_features -> h_size, n_layers, bidirectional?,
batch_first)`` -> ``Linear(h*dirs -> h)`` -> ``Linear(h -> 64)`` -> ``Linear(64 -> 1)`` with
NO activations between the linears (app/torch_train.py:199-205); fresh random ``(h0, c0)``
every forward (app/torch_train.py:179-193); the last timestep is selected
(app/torch_train.py:196); output shape ``[B, 1, 1]``.  ``state_dict`` keys are identical to
the reference's (``lstm.weight_ih_l0`` … ``linear3.bias``) so ``broadcast_parameters``
moves the same 10 tensors / 1 480 196 bytes.

H100-first changes (SURVEY.md §2.6 S2/S4, §7.3):
  * ``(h0, c0)`` come from the device generator (no CPU randn + pageable H2D + sync per
    step), the last-step gather is a slice (no host-built index tensor);
  * on CUDA (fp32, hidden size 256, one unidirectional layer — the reference configuration)
    forward/backward run on the persistent cluster LSTM kernels (K5: ``ops/lstm_rec.py``,
    csrc/lstm_rec_sm90.cu — tf32 wgmma, W_hh resident in shared memory, h exchanged through
    DSMEM) and the chained-GEMM head (K6: ``ops/lstm_fused.py``); other shapes (bidirectional,
    multi-layer, other hidden sizes) use cuDNN / cuBLAS, which is also the numerics oracle.
"""
from __future__ import annotations

import warnings
from typing import Callable, Optional, Sequence

import torch
from torch import nn


class LSTM(nn.Module):
    """implements an lstm - a single/multilayer uni/bi directional lstm"""

    def __init__(self, n_features, window_size, output_size, h_size, n_layers=1,
                 bidirectional=False, device=torch.device('cpu'),
                 initializers: Optional[Sequence[Callable]] = None, fused: Optional[bool] = None):
        super().__init__()
        self.n_features = n_features
        self.window_size = window_size
        self.output_size = output_size
        self.h_size = h_size
        self.n_layers = n_layers
        self.directions = 2 if bidirectional else 1
        self.device = torch.device(device)

        self.lstm = nn.LSTM(input_size=n_features, hidden_size=h_size, num_layers=n_layers,
                            bidirectional=bidirectional, batch_first=True)
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

    def _use_fused(self, x: torch.Tensor) -> bool:
        if self._fused is False or not x.is_cuda:
            return False
        if self.directions != 1:
            return False
        from ..ops import lstm_fused
        return lstm_fused.available(self, x)

    def forward(self, input):
        batch_size = input.size(0)
        self.hidden = self.init_hidden(batch_size)
        if self._use_fused(input):
            from ..ops import lstm_fused
            return lstm_fused.forward(self, input, self.hidden)
        lstm_output, self.hidden = self.lstm(input, self.hidden)
        last_hidden_states = lstm_output[:, self.window_size - 1:self.window_size, :]
        return self.linear3(self.linear2(self.linear(last_hidden_states)))
