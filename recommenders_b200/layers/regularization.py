"""`Dropout` and `SpatialDropout1D`: tf.keras's dropout layers on K23.  DESIGN.md §2 (A26) pins the mask rule."""
from __future__ import annotations

from typing import Any, Dict

import torch

from .. import ops
from ..backend import resolve_training


class Dropout(torch.nn.Module):
  """`tf.keras.layers.Dropout(rate, noise_shape=None, seed=None)`.  In training y = keep ? x / (1 - rate) : +0, each
  element kept with probability 1 - rate; at inference (and at rate 0) the input is returned as is, with no launch.
  `training` resolves as `backend.resolve_training` says: the argument, then the innermost learning-phase scope
  (`Model.train_step` opens a training one), then False.

  The mask is Philox4x32-10 keyed by the layer's 64-bit seed; `seed=None` draws the key once, at construction, from
  torch's default CPU generator, so `torch.manual_seed` makes runs reproducible.  A per-layer call counter, advanced
  once per training call, is the Philox counter's high half, so successive calls draw different masks.  `noise_shape`
  follows Keras: a None entry takes the input's size, a size-1 entry broadcasts one mask value along that axis.  Inputs
  are float32 CUDA tensors of rank 1 to 4.  A mask attached by `Embedding(mask_zero=True)` is attached to the output."""

  def __init__(self, rate: float, noise_shape=None, seed=None, name=None, **kwargs):
    super().__init__()
    if isinstance(rate, (int, float)) and not 0 <= rate < 1:
      raise ValueError(f"Invalid value received for argument `rate`. Expected a float value between 0 and 1. "
                       f"Received: rate={rate}")
    self.rate = float(rate)
    self.noise_shape = None if noise_shape is None else tuple(noise_shape)
    self.seed = seed
    if seed is None:
      lo, hi = torch.randint(0, 2**32, (2,), dtype=torch.int64).tolist()
      self._key = lo | (hi << 32)
    else:
      self._key = int(seed) & (2**64 - 1)
    self._calls = 0
    self.name = name

  def _noise_shape(self, inputs: torch.Tensor):
    return self.noise_shape

  def call(self, inputs: torch.Tensor, training=None):
    if not isinstance(inputs, torch.Tensor):
      raise TypeError(f"{type(self).__name__}: inputs must be a torch.Tensor, got {type(inputs)}")
    noise = self._noise_shape(inputs)
    if not resolve_training(training) or self.rate == 0.0:
      return inputs
    mask = ops.attached_mask(inputs)
    call = self._calls
    self._calls += 1
    return ops.attach_mask(ops.dropout(inputs, self.rate, self._key, call, noise), mask)

  def forward(self, inputs, training=None):
    return self.call(inputs, training=training)

  def get_config(self) -> Dict[str, Any]:
    return {"rate": self.rate, "noise_shape": self.noise_shape, "seed": self.seed, "name": self.name}

  @classmethod
  def from_config(cls, config: Dict[str, Any]):
    return cls(**config)


class SpatialDropout1D(Dropout):
  """`tf.keras.layers.SpatialDropout1D(rate, seed=None)`: Dropout with noise_shape (B, 1, D), so a whole feature
  channel of a [B, T, D] sequence is dropped or kept for all its steps.  A non-3-D input raises ValueError."""

  def __init__(self, rate: float, seed=None, name=None, **kwargs):
    super().__init__(rate, seed=seed, name=name)

  def _noise_shape(self, inputs: torch.Tensor):
    if inputs.dim() != 3:
      raise ValueError(f"SpatialDropout1D: the input must be 3-D [B, T, D], got shape {tuple(inputs.shape)}")
    return (inputs.shape[0], 1, inputs.shape[2])

  def get_config(self) -> Dict[str, Any]:
    return {"rate": self.rate, "seed": self.seed, "name": self.name}
