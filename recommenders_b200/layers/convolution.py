"""`Conv1D`, the layer of convolutional sequence towers: NextItNet-style next-item towers (stacks of causal, dilated
convolutions with residual connections) and text-CNN title encoders.  tf.keras.layers.Conv1D (channels_last, groups = 1)
on K27, DESIGN.md §2 (A29)."""
from __future__ import annotations

from typing import Any, Dict

import numpy as np
import torch

from .. import ops
from .attention import _kernel_init
from .blocks import _activation_name
from .feature_interaction.dcn import _ACTIVATIONS, _init


def _normalize_tuple(value, name: str, allow_zero: bool = False):
  """tf-keras `conv_utils.normalize_tuple` for rank 1: an int or a one-int sequence, > 0 (>= 0 with allow_zero)."""
  msg = f"The `{name}` argument must be a tuple of 1 integers. Received {name}={value}"
  if isinstance(value, (int, np.integer)) and not isinstance(value, bool):
    t = (int(value),)
  else:
    try:
      t = tuple(value)
    except TypeError:
      raise ValueError(msg) from None
    if len(t) != 1 or isinstance(t[0], bool) or not isinstance(t[0], (int, np.integer)):
      raise ValueError(msg)
    t = (int(t[0]),)
  bad = {v for v in t if (v < 0 if allow_zero else v <= 0)}
  if bad:
    raise ValueError(f"{msg} including values {bad} that do not satisfy the requirement `{'>= 0' if allow_zero else '> 0'}`.")
  return t


class Conv1D(torch.nn.Module):
  """`tf.keras.layers.Conv1D(filters, kernel_size, strides, padding, dilation_rate, activation, use_bias, ...)`: x [B, T, C]
  float32 -> [B, T_out, filters] with y[b, t, n] = act(bias[n] + sum_j sum_c x[b, t s + j d - p, c] kernel[j, c, n]),
  positions outside [0, T) reading 0.  padding "valid" (p = 0), "same" (T_out = ceil(T / s), the extra pad column on the
  right) or "causal" (p = d (k - 1)); `ops.conv1d_geometry` gives T_out and p.  Weights as Keras stores them, created on
  the first call: kernel [k, C, filters] ("glorot_uniform" with Keras's fans for a rank-3 kernel), bias [filters].

  linear / relu / sigmoid run fused in K27 (tensor cores at large shapes, the exact fmaf chain otherwise); any other
  activation of `dcn._ACTIVATIONS`, or a callable, is applied to the fused linear output.  Keras's argument errors are
  raised as Keras raises them; groups > 1, channels_first, regularizers, constraints and inputs of rank other than 3 raise
  NotImplementedError.  Conv1D does not support masking: an input that carries a Keras mask raises TypeError, as tf-keras's
  base `compute_mask` does."""

  def __init__(self, filters: int, kernel_size, strides=1, padding: str = "valid", data_format: str = "channels_last",
               dilation_rate=1, groups: int = 1, activation=None, use_bias: bool = True, kernel_initializer="glorot_uniform",
               bias_initializer="zeros", kernel_regularizer=None, bias_regularizer=None, activity_regularizer=None,
               kernel_constraint=None, bias_constraint=None, name=None, **kwargs):
    super().__init__()
    if isinstance(filters, float):
      filters = int(filters)
    if isinstance(filters, bool) or not isinstance(filters, (int, np.integer)) or filters <= 0:
      raise ValueError(f"Invalid value for argument `filters`. Expected a strictly positive value. Received filters={filters}.")
    self.filters = int(filters)
    self.kernel_size = _normalize_tuple(kernel_size, "kernel_size")
    self.strides = _normalize_tuple(strides, "strides", allow_zero=True)
    pad = padding.lower() if isinstance(padding, str) else padding
    if pad not in ops.CONV1D_PADDINGS:
      raise ValueError(f'The `padding` argument must be a list/tuple or one of "valid", "same" (or "causal", only for '
                       f"`Conv1D). Received: {padding}")
    self.padding = pad
    fmt = data_format.lower() if isinstance(data_format, str) else data_format
    if fmt not in ("channels_last", "channels_first"):
      raise ValueError(f'The `data_format` argument must be one of "channels_first", "channels_last". Received: {data_format}')
    self.dilation_rate = _normalize_tuple(dilation_rate, "dilation_rate")
    if isinstance(groups, bool) or not isinstance(groups, (int, np.integer)) or groups <= 0:
      raise ValueError(f"The number of groups must be a positive integer. Received: groups={groups}.")
    if self.filters % groups != 0:
      raise ValueError(f"The number of filters must be evenly divisible by the number of groups. Received: groups={groups}, "
                       f"filters={filters}.")
    if not all(self.strides):
      raise ValueError(f"The argument `strides` cannot contains 0(s). Received: {self.strides}")
    if max(self.strides) > 1 and max(self.dilation_rate) > 1:
      raise ValueError(f"`strides > 1` not supported in conjunction with `dilation_rate > 1`. Received: "
                       f"strides={self.strides} and dilation_rate={self.dilation_rate}")
    if isinstance(activation, str) and activation not in _ACTIVATIONS:
      raise ValueError(f"Unknown activation function: {activation}")
    unsupported = {
        "groups": groups != 1,
        "data_format": fmt != "channels_last",
        "kernel_regularizer": kernel_regularizer is not None,
        "bias_regularizer": bias_regularizer is not None,
        "activity_regularizer": activity_regularizer is not None,
        "kernel_constraint": kernel_constraint is not None,
        "bias_constraint": bias_constraint is not None,
    }
    for arg, bad in unsupported.items():
      if bad:
        raise NotImplementedError(f"Conv1D: {arg}={locals()[arg]!r} is not supported")
    self.data_format, self.groups = fmt, 1
    self._activation_cfg = activation
    self.use_bias = bool(use_bias)
    self._kernel_initializer = kernel_initializer
    self._bias_initializer = bias_initializer
    self.name = name
    self.built = False

  def build(self, input_shape, device=None):
    C = int(input_shape[-1])
    device = device or torch.device("cuda", torch.cuda.current_device())
    self.kernel = torch.nn.Parameter(_kernel_init(self._kernel_initializer, (self.kernel_size[0], C, self.filters), device))
    self.bias = torch.nn.Parameter(_init(self._bias_initializer, (self.filters,), device)) if self.use_bias else None
    self.built = True

  def compute_mask(self, inputs, mask=None):
    """tf-keras's base `Layer.compute_mask` for a layer without masking support: any mask raises TypeError."""
    if mask is not None:
      raise TypeError(f"Layer {self.name or 'conv1d'} does not support masking, but was passed an input_mask: {mask}")
    return None

  def call(self, inputs: torch.Tensor, mask=None) -> torch.Tensor:
    if isinstance(inputs, torch.Tensor) and inputs.dim() != 3:
      raise NotImplementedError(f"Conv1D: inputs of rank {inputs.dim()} are not supported (expected [batch, steps, channels])")
    self.compute_mask(inputs, ops.layer_mask(inputs, mask))
    if not self.built:
      self.build(inputs.shape, inputs.device if isinstance(inputs, torch.Tensor) else None)
    a = self._activation_cfg
    args = (inputs, self.kernel, self.bias, self.strides[0], self.padding, self.dilation_rate[0])
    if a is None or (isinstance(a, str) and a in ops.DENSE_ACTIVATIONS):
      return ops.conv1d(*args, activation=a)
    fn = _ACTIVATIONS[a] if isinstance(a, str) else a
    return fn(ops.conv1d(*args, activation=None))

  def forward(self, inputs, mask=None):
    return self.call(inputs, mask=mask)

  def get_config(self) -> Dict[str, Any]:
    init = lambda i: i if isinstance(i, str) else "custom"
    return {"filters": self.filters, "kernel_size": self.kernel_size, "strides": self.strides, "padding": self.padding,
            "data_format": self.data_format, "dilation_rate": self.dilation_rate, "groups": self.groups,
            "activation": _activation_name(self._activation_cfg), "use_bias": self.use_bias,
            "kernel_initializer": init(self._kernel_initializer), "bias_initializer": init(self._bias_initializer),
            "kernel_regularizer": None, "bias_regularizer": None, "activity_regularizer": None, "kernel_constraint": None,
            "bias_constraint": None, "name": self.name}

  @classmethod
  def from_config(cls, config: Dict[str, Any]):
    return cls(**config)
