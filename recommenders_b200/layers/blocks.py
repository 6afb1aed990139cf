"""Dense blocks: mirror of tensorflow_recommenders/layers/blocks.py (MLP), with `Dense` standing in for
tf.keras.layers.Dense, which the reference's MLP and the tutorials' ranking towers are built from."""
from __future__ import annotations

from typing import Callable, List, Optional, Union

import torch

from .. import ops
from .feature_interaction.dcn import _ACTIVATIONS, _init

Activation = Union[None, str, Callable]


def _activation_name(a: Activation):
  return a if (a is None or isinstance(a, str)) else getattr(a, "__name__", str(a))


class Dense(torch.nn.Module):
  """`tf.keras.layers.Dense(units, activation, use_bias, kernel_initializer, bias_initializer)`:  act(x @ kernel + bias),
  kernel [in, units].  Weights are created on the first call (Keras `build`).

  linear / relu / sigmoid run fused in the K6 kernels (tensor cores at large shapes, the exact fmaf chain otherwise);
  any other activation of `dcn._ACTIVATIONS`, or a callable, is applied to the fused linear output."""

  def __init__(self, units: int, activation: Activation = None, use_bias: bool = True,
               kernel_initializer="glorot_uniform", bias_initializer="zeros", name: Optional[str] = None, **kwargs):
    super().__init__()
    self.units = int(units)
    if self.units <= 0:
      raise ValueError(f"Received an invalid value for `units`, expected a positive integer. Received: units={units}")
    if isinstance(activation, str) and activation not in _ACTIVATIONS:
      raise ValueError(f"Unknown activation function: {activation}")
    self._activation_cfg = activation
    self.use_bias = use_bias
    self._kernel_initializer = kernel_initializer
    self._bias_initializer = bias_initializer
    self.name = name
    self.built = False

  def build(self, input_shape, device=None):
    last_dim = int(input_shape[-1])
    device = device or torch.device("cuda", torch.cuda.current_device())
    self.kernel = torch.nn.Parameter(_init(self._kernel_initializer, (last_dim, self.units), device))
    self.bias = torch.nn.Parameter(_init(self._bias_initializer, (self.units,), device)) if self.use_bias else None
    self.built = True

  def call(self, x: torch.Tensor) -> torch.Tensor:
    if not self.built:
      self.build(x.shape, x.device if isinstance(x, torch.Tensor) else None)
    a = self._activation_cfg
    if a is None or (isinstance(a, str) and a in ops.DENSE_ACTIVATIONS):
      return ops.dense(x, self.kernel, self.bias, a)
    fn = _ACTIVATIONS[a] if isinstance(a, str) else a
    return fn(ops.dense(x, self.kernel, self.bias, None))

  def forward(self, x):
    return self.call(x)

  def get_config(self):
    return {
        "units": self.units,
        "activation": _activation_name(self._activation_cfg),
        "use_bias": self.use_bias,
        "kernel_initializer": self._kernel_initializer if isinstance(self._kernel_initializer, str) else "custom",
        "bias_initializer": self._bias_initializer if isinstance(self._bias_initializer, str) else "custom",
        "name": self.name,
    }

  @classmethod
  def from_config(cls, config):
    return cls(**config)


class MLP(torch.nn.Module):
  """Sequential multi-layer perceptron (MLP) block (blocks.py:24-61): `Dense(n, activation)` for every size but the last,
  `Dense(units[-1], final_activation)` last."""

  def __init__(self, units: List[int], use_bias: bool = True, activation: Activation = "relu",
               final_activation: Activation = None, **kwargs) -> None:
    super().__init__()
    self._units = list(units)
    self._use_bias = use_bias
    self._activation = activation
    self._final_activation = final_activation
    self.name = kwargs.get("name")
    layers = [Dense(n, activation=activation, use_bias=use_bias) for n in self._units[:-1]]
    layers.append(Dense(self._units[-1], activation=final_activation, use_bias=use_bias))
    self._sublayers = torch.nn.ModuleList(layers)

  def call(self, x: torch.Tensor) -> torch.Tensor:
    for layer in self._sublayers:
      x = layer(x)
    return x

  def forward(self, x):
    return self.call(x)

  def get_config(self):
    return {"units": list(self._units), "use_bias": self._use_bias, "activation": _activation_name(self._activation),
            "final_activation": _activation_name(self._final_activation), "name": self.name}

  @classmethod
  def from_config(cls, config):
    return cls(**config)
