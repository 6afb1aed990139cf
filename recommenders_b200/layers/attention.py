"""`MultiHeadAttention`, the self-attention block of SASRec-style query towers and of the Transformer title encoders the
featurization tutorial points to: tf.keras.layers.MultiHeadAttention on K6 (the four projections) and K21 (the
attention core).  DESIGN.md §2 (A25) pins its rules."""
from __future__ import annotations

import math
from typing import Any, Dict

import numpy as np
import torch

from .. import ops
from .feature_interaction.dcn import _init


def keras_fans(shape):
  """tf-keras `_compute_fans`: for a kernel of rank > 2 the leading dimensions are a receptive field, fan_in =
  shape[-2] * prod(shape[:-2]) and fan_out = shape[-1] * prod(shape[:-2])."""
  if len(shape) == 0:
    return 1, 1
  if len(shape) == 1:
    return shape[0], shape[0]
  field = math.prod(shape[:-2])
  return shape[-2] * field, shape[-1] * field


def _kernel_init(name, shape, device):
  if name == "glorot_uniform":
    fan_in, fan_out = keras_fans(shape)
    limit = math.sqrt(6.0 / (fan_in + fan_out))
    return torch.empty(shape, dtype=torch.float32, device=device).uniform_(-limit, limit)
  return _init(name, shape, device)


class _Projection(torch.nn.Module):
  """The weights of one of Keras's EinsumDense sublayers, so that they appear as `query.kernel`, `query.bias`, ..."""

  def __init__(self, kernel: torch.Tensor, bias):
    super().__init__()
    self.kernel = torch.nn.Parameter(kernel)
    self.bias = None if bias is None else torch.nn.Parameter(bias)


def _as_mask(mask, device):
  if mask is None or isinstance(mask, torch.Tensor):
    return mask
  return torch.from_numpy(np.ascontiguousarray(mask)).to(device)


class MultiHeadAttention(torch.nn.Module):
  """`tf.keras.layers.MultiHeadAttention(num_heads, key_dim)`: `layer(query, value, key=None)` with query [B, T, D_q],
  value [B, S, D_v], key [B, S, D_k] (key = value when None) -> [B, T, D_out] (D_out = D_q unless `output_shape`), and
  with `return_attention_scores` also the softmax scores [B, H, T, S], returned detached: they carry no gradient.

  Weights as Keras stores them, created on the first call: query.kernel [D_q, H, dk], key.kernel [D_k, H, dk],
  value.kernel [D_v, H, dv], attention_output.kernel [H, dv, D_out], biases [H, dk] / [H, dk] / [H, dv] / [D_out];
  "glorot_uniform" uses Keras's fans for these 3-D kernels.  Masks combine as Keras's `_compute_attention_mask`:
  query_mask [B, T], value_mask [B, S], key_mask [B, S] (each passed, or attached to the input by an
  `Embedding(mask_zero=True)`), the causal triangle with `use_causal_mask`, and `attention_mask` [B, T, S]; a dropped
  score gets -1e9, so a fully masked row attends uniformly.  The output carries the query's mask.

  key_dim and value_dim go up to 128 (ops.MHA_MAX_HEAD_DIM).  attention_axes other than the sequence axis, dropout,
  regularizers, constraints and inputs of rank other than 3 raise NotImplementedError."""

  def __init__(self, num_heads: int, key_dim: int, value_dim=None, dropout: float = 0.0, use_bias: bool = True,
               output_shape=None, attention_axes=None, kernel_initializer="glorot_uniform", bias_initializer="zeros",
               kernel_regularizer=None, bias_regularizer=None, activity_regularizer=None, kernel_constraint=None,
               bias_constraint=None, name=None, **kwargs):
    super().__init__()
    for arg, val in (("num_heads", num_heads), ("key_dim", key_dim), ("value_dim", value_dim)):
      if val is None and arg == "value_dim":
        continue
      if isinstance(val, bool) or not isinstance(val, (int, np.integer)) or val <= 0:
        raise ValueError(f"MultiHeadAttention: {arg} must be a positive integer, got {val!r}")
    value_dim = key_dim if value_dim is None else value_dim
    for arg, val in (("key_dim", key_dim), ("value_dim", value_dim)):
      if val > ops.MHA_MAX_HEAD_DIM:
        raise ValueError(f"MultiHeadAttention: {arg} = {val} is above the kernel's ceiling of {ops.MHA_MAX_HEAD_DIM}")
    axes = attention_axes
    if isinstance(axes, (list, tuple)) and len(axes) == 1:
      axes = axes[0]
    unsupported = {
        "attention_axes": axes not in (None, 1, -2),
        "dropout": dropout != 0,
        "kernel_regularizer": kernel_regularizer is not None,
        "bias_regularizer": bias_regularizer is not None,
        "activity_regularizer": activity_regularizer is not None,
        "kernel_constraint": kernel_constraint is not None,
        "bias_constraint": bias_constraint is not None,
    }
    for arg, bad in unsupported.items():
      if bad:
        raise NotImplementedError(f"MultiHeadAttention: {arg}={locals()[arg]!r} is not supported")
    if output_shape is not None:
      shape = tuple(output_shape) if isinstance(output_shape, (list, tuple)) else (output_shape,)
      if len(shape) != 1:
        raise NotImplementedError(f"MultiHeadAttention: output_shape={output_shape!r} (more than one axis) is not "
                                  "supported")
    self.num_heads, self.key_dim, self.value_dim = int(num_heads), int(key_dim), int(value_dim)
    self.dropout, self.use_bias = float(dropout), bool(use_bias)
    self.output_shape, self.attention_axes = output_shape, attention_axes
    self._kernel_initializer, self._bias_initializer = kernel_initializer, bias_initializer
    self.name = name
    self.built = False

  def build(self, query_shape, value_shape, key_shape=None, device=None):
    key_shape = value_shape if key_shape is None else key_shape
    device = device or torch.device("cuda", torch.cuda.current_device())
    H, dk, dv = self.num_heads, self.key_dim, self.value_dim
    if self.output_shape is None:
      d_out = int(query_shape[-1])
    else:
      d_out = int(self.output_shape[0] if isinstance(self.output_shape, (list, tuple)) else self.output_shape)
    bias = lambda shape: _init(self._bias_initializer, shape, device) if self.use_bias else None
    self.query = _Projection(_kernel_init(self._kernel_initializer, (int(query_shape[-1]), H, dk), device), bias((H, dk)))
    self.key = _Projection(_kernel_init(self._kernel_initializer, (int(key_shape[-1]), H, dk), device), bias((H, dk)))
    self.value = _Projection(_kernel_init(self._kernel_initializer, (int(value_shape[-1]), H, dv), device),
                             bias((H, dv)))
    self.attention_output = _Projection(_kernel_init(self._kernel_initializer, (H, dv, d_out), device), bias((d_out,)))
    self.built = True

  def call(self, query, value, key=None, attention_mask=None, return_attention_scores: bool = False, training=None,
           use_causal_mask: bool = False, query_mask=None, value_mask=None, key_mask=None):
    for t, name in ((query, "query"), (value, "value"), (key, "key")):
      if t is not None and (not isinstance(t, torch.Tensor) or t.dim() != 3):
        rank = t.dim() if isinstance(t, torch.Tensor) else None
        raise NotImplementedError(f"MultiHeadAttention: {name} of rank {rank} is not supported (rank 3 only)")
    if not self.built:
      self.build(query.shape, value.shape, None if key is None else key.shape, query.device)
    dev = query.device
    query_mask = ops.attached_mask(query) if query_mask is None else _as_mask(query_mask, dev)
    value_mask = ops.attached_mask(value) if value_mask is None else _as_mask(value_mask, dev)
    if key_mask is None and key is not None:
      key_mask = ops.attached_mask(key)
    key_mask = _as_mask(key_mask, dev)
    attention_mask = _as_mask(attention_mask, dev)
    p = (self.query, self.key, self.value, self.attention_output)
    out, scores = ops.attention(query, value, key, *(w.kernel for w in p), *(w.bias for w in p), query_mask=query_mask,
                                value_mask=value_mask, key_mask=key_mask, attention_mask=attention_mask,
                                causal=bool(use_causal_mask), return_scores=bool(return_attention_scores))
    if query_mask is not None:
      out._tfrs_mask = (query_mask, out._version, out.data_ptr())
    return (out, scores) if return_attention_scores else out

  def forward(self, query, value, key=None, attention_mask=None, return_attention_scores: bool = False, training=None,
              use_causal_mask: bool = False, query_mask=None, value_mask=None, key_mask=None):
    return self.call(query, value, key, attention_mask=attention_mask, return_attention_scores=return_attention_scores,
                     training=training, use_causal_mask=use_causal_mask, query_mask=query_mask, value_mask=value_mask,
                     key_mask=key_mask)

  def get_config(self) -> Dict[str, Any]:
    return {"num_heads": self.num_heads, "key_dim": self.key_dim, "value_dim": self.value_dim, "dropout": self.dropout,
            "use_bias": self.use_bias, "output_shape": self.output_shape, "attention_axes": self.attention_axes,
            "kernel_initializer": self._kernel_initializer, "bias_initializer": self._bias_initializer,
            "kernel_regularizer": None, "bias_regularizer": None, "activity_regularizer": None,
            "kernel_constraint": None, "bias_constraint": None, "name": self.name}

  @classmethod
  def from_config(cls, config: Dict[str, Any]):
    return cls(**config)
