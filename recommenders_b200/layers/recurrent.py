"""`GRU`, the query tower of the reference's sequential retrieval tutorial (`Sequential([StringLookup, Embedding,
GRU(32)])`): tf.keras.layers.GRU with the TF2 defaults (reset_after=True) on K6 (the input projection) and K19 (the
recurrence).  `LSTM`, the cell often put in that tower instead: tf.keras.layers.LSTM on K6 and K20.  DESIGN.md §2 (A23,
A24) pins their rules."""
from __future__ import annotations

from typing import Any, Dict

import numpy as np
import torch

from .. import ops
from .feature_interaction.dcn import _init


class GRU(torch.nn.Module):
  """`tf.keras.layers.GRU(units)`: x [B, T, D] float32 -> h_T [B, units], or every h_t [B, T, units] with
  `return_sequences`; `return_state` returns Keras's `[output, h_T]`.  Weights as Keras stores them, created on the first
  call: kernel [D, 3u], recurrent_kernel [u, 3u], bias [2, 3u] (input and recurrent bias), columns (z, r, h).  A mask
  ([B, T] bool or int ids, nonzero = kept; passed as `mask=` or carried by an `Embedding(mask_zero=True)` output) carries
  the state unchanged through masked steps, so an all-masked row returns its initial state.

  Keras's tanh / sigmoid activations with reset_after=True are what the kernels compute; another activation,
  reset_after=False, dropout, go_backwards, stateful, time_major, and a mask with return_sequences=True (where Keras's
  cuDNN and generic paths disagree on the outputs at masked steps) raise NotImplementedError.  `unroll` changes nothing:
  every sequence runs as one kernel launch."""

  def __init__(self, units: int, activation="tanh", recurrent_activation="sigmoid", use_bias: bool = True,
               kernel_initializer="glorot_uniform", recurrent_initializer="orthogonal", bias_initializer="zeros",
               dropout: float = 0.0, recurrent_dropout: float = 0.0, return_sequences: bool = False,
               return_state: bool = False, go_backwards: bool = False, stateful: bool = False, unroll: bool = False,
               time_major: bool = False, reset_after: bool = True, name=None, **kwargs):
    super().__init__()
    if isinstance(units, bool) or not isinstance(units, (int, np.integer)) or units <= 0:
      raise ValueError(f"Received an invalid value for argument `units`, expected a positive integer, got {units}.")
    if units > ops.GRU_MAX_UNITS:
      raise ValueError(f"GRU: units = {units} is above the kernel's ceiling of {ops.GRU_MAX_UNITS}")
    unsupported = {
        "activation": activation not in ("tanh", torch.tanh),
        "recurrent_activation": recurrent_activation not in ("sigmoid", torch.sigmoid),
        "reset_after": not reset_after,
        "dropout": dropout != 0,
        "recurrent_dropout": recurrent_dropout != 0,
        "go_backwards": bool(go_backwards),
        "stateful": bool(stateful),
        "time_major": bool(time_major),
    }
    for arg, bad in unsupported.items():
      if bad:
        raise NotImplementedError(f"GRU: {arg}={locals()[arg]!r} is not supported")
    self.units = int(units)
    self.use_bias = bool(use_bias)
    self.return_sequences, self.return_state, self.unroll = bool(return_sequences), bool(return_state), bool(unroll)
    self._kernel_initializer = kernel_initializer
    self._recurrent_initializer = recurrent_initializer
    self._bias_initializer = bias_initializer
    self.name = name
    self.built = False

  def build(self, input_shape, device=None):
    D, u = int(input_shape[-1]), self.units
    device = device or torch.device("cuda", torch.cuda.current_device())
    self.kernel = torch.nn.Parameter(_init(self._kernel_initializer, (D, 3 * u), device))
    self.recurrent_kernel = torch.nn.Parameter(_init(self._recurrent_initializer, (u, 3 * u), device))
    self.bias = torch.nn.Parameter(_init(self._bias_initializer, (2, 3 * u), device)) if self.use_bias else None
    self.built = True

  def call(self, inputs: torch.Tensor, mask=None, training=None, initial_state=None):
    if not self.built:
      self.build(inputs.shape, inputs.device if isinstance(inputs, torch.Tensor) else None)
    mask = ops.layer_mask(inputs, mask)
    if isinstance(initial_state, (list, tuple)):
      if len(initial_state) != 1:
        raise ValueError(f"GRU: expected one initial state, got {len(initial_state)}")
      initial_state = initial_state[0]
    out, h = ops.gru(inputs, self.kernel, self.recurrent_kernel, self.bias, initial_state, mask, self.return_sequences)
    return [out, h] if self.return_state else out

  def forward(self, inputs, mask=None, training=None, initial_state=None):
    return self.call(inputs, mask=mask, training=training, initial_state=initial_state)

  def get_config(self) -> Dict[str, Any]:
    return {"units": self.units, "activation": "tanh", "recurrent_activation": "sigmoid", "use_bias": self.use_bias,
            "kernel_initializer": self._kernel_initializer, "recurrent_initializer": self._recurrent_initializer,
            "bias_initializer": self._bias_initializer, "dropout": 0.0, "recurrent_dropout": 0.0,
            "return_sequences": self.return_sequences, "return_state": self.return_state, "go_backwards": False,
            "stateful": False, "unroll": self.unroll, "time_major": False, "reset_after": True, "name": self.name}

  @classmethod
  def from_config(cls, config: Dict[str, Any]):
    return cls(**config)


class LSTM(torch.nn.Module):
  """`tf.keras.layers.LSTM(units)`: x [B, T, D] float32 -> h_T [B, units], or every h_t [B, T, units] with
  `return_sequences`; `return_state` returns Keras's `[output, h_T, c_T]`, and `initial_state` takes `[h_0, c_0]`.
  Weights as Keras stores them, created on the first call: kernel [D, 4u], recurrent_kernel [u, 4u], bias [4u], columns
  (i, f, c, o).  With `unit_forget_bias` (the default) the forget slice bias[u:2u] starts at 1 and the other slices
  come from `bias_initializer`.  A mask ([B, T] bool or int ids, nonzero = kept; passed as `mask=` or carried by an
  `Embedding(mask_zero=True)` output) carries h and c unchanged through masked steps, so an all-masked row returns its
  initial state.

  Keras's tanh / sigmoid activations are what the kernels compute; another activation, dropout, go_backwards, stateful,
  time_major, and a mask with return_sequences=True (where Keras's cuDNN and generic paths disagree on the outputs at
  masked steps) raise NotImplementedError.  `implementation` and `unroll` change nothing: every sequence runs as one
  kernel launch (K6 for the projection, K20 for the recurrence)."""

  def __init__(self, units: int, activation="tanh", recurrent_activation="sigmoid", use_bias: bool = True,
               kernel_initializer="glorot_uniform", recurrent_initializer="orthogonal", bias_initializer="zeros",
               unit_forget_bias: bool = True, dropout: float = 0.0, recurrent_dropout: float = 0.0,
               return_sequences: bool = False, return_state: bool = False, go_backwards: bool = False,
               stateful: bool = False, time_major: bool = False, unroll: bool = False, implementation: int = 2,
               name=None, **kwargs):
    super().__init__()
    if isinstance(units, bool) or not isinstance(units, (int, np.integer)) or units <= 0:
      raise ValueError(f"Received an invalid value for argument `units`, expected a positive integer, got {units}.")
    if units > ops.LSTM_MAX_UNITS:
      raise ValueError(f"LSTM: units = {units} is above the kernel's ceiling of {ops.LSTM_MAX_UNITS}")
    unsupported = {
        "activation": activation not in ("tanh", torch.tanh),
        "recurrent_activation": recurrent_activation not in ("sigmoid", torch.sigmoid),
        "dropout": dropout != 0,
        "recurrent_dropout": recurrent_dropout != 0,
        "go_backwards": bool(go_backwards),
        "stateful": bool(stateful),
        "time_major": bool(time_major),
    }
    for arg, bad in unsupported.items():
      if bad:
        raise NotImplementedError(f"LSTM: {arg}={locals()[arg]!r} is not supported")
    self.units = int(units)
    self.use_bias, self.unit_forget_bias = bool(use_bias), bool(unit_forget_bias)
    self.return_sequences, self.return_state, self.unroll = bool(return_sequences), bool(return_state), bool(unroll)
    self.implementation = implementation
    self._kernel_initializer = kernel_initializer
    self._recurrent_initializer = recurrent_initializer
    self._bias_initializer = bias_initializer
    self.name = name
    self.built = False

  def build(self, input_shape, device=None):
    D, u = int(input_shape[-1]), self.units
    device = device or torch.device("cuda", torch.cuda.current_device())
    self.kernel = torch.nn.Parameter(_init(self._kernel_initializer, (D, 4 * u), device))
    self.recurrent_kernel = torch.nn.Parameter(_init(self._recurrent_initializer, (u, 4 * u), device))
    self.bias = None
    if self.use_bias:
      if self.unit_forget_bias:   # Keras: concat(bias_initializer(u), ones(u), bias_initializer(2u))
        b = torch.cat([_init(self._bias_initializer, (u,), device), torch.ones(u, device=device),
                       _init(self._bias_initializer, (2 * u,), device)]).contiguous()
      else:
        b = _init(self._bias_initializer, (4 * u,), device)
      self.bias = torch.nn.Parameter(b)
    self.built = True

  def call(self, inputs: torch.Tensor, mask=None, training=None, initial_state=None):
    if not self.built:
      self.build(inputs.shape, inputs.device if isinstance(inputs, torch.Tensor) else None)
    mask = ops.layer_mask(inputs, mask)
    if initial_state is not None and (isinstance(initial_state, torch.Tensor) or len(initial_state) != 2):
      n = 1 if isinstance(initial_state, torch.Tensor) else len(initial_state)
      raise ValueError(f"LSTM: expected two initial states [h_0, c_0], got {n}")
    out, h, c = ops.lstm(inputs, self.kernel, self.recurrent_kernel, self.bias, initial_state, mask,
                         self.return_sequences)
    return [out, h, c] if self.return_state else out

  def forward(self, inputs, mask=None, training=None, initial_state=None):
    return self.call(inputs, mask=mask, training=training, initial_state=initial_state)

  def get_config(self) -> Dict[str, Any]:
    return {"units": self.units, "activation": "tanh", "recurrent_activation": "sigmoid", "use_bias": self.use_bias,
            "kernel_initializer": self._kernel_initializer, "recurrent_initializer": self._recurrent_initializer,
            "bias_initializer": self._bias_initializer, "unit_forget_bias": self.unit_forget_bias, "dropout": 0.0,
            "recurrent_dropout": 0.0, "return_sequences": self.return_sequences, "return_state": self.return_state,
            "go_backwards": False, "stateful": False, "time_major": False, "unroll": self.unroll,
            "implementation": self.implementation, "name": self.name}

  @classmethod
  def from_config(cls, config: Dict[str, Any]):
    return cls(**config)
