"""`MultiHeadAttention`, `Attention` and `AdditiveAttention`.  MultiHeadAttention is the self-attention block of
SASRec-style query towers and of the Transformer title encoders the featurization tutorial points to:
tf.keras.layers.MultiHeadAttention on K6 (the four projections) and K21 (the attention core), DESIGN.md §2 (A25).  Attention and AdditiveAttention are the target attention of DIN / BST-style
ranking models (a candidate attending over a user's history): tf.keras's dense attention layers on K21's dot scores and
K25's tanh scores, DESIGN.md §2 (A27)."""
from __future__ import annotations

import math
from typing import Any, Dict

import numpy as np
import torch

from .. import ops
from ..backend import resolve_training
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
    query_mask = ops.layer_mask(query, query_mask)
    value_mask = ops.layer_mask(value, value_mask)
    if key is not None or key_mask is not None:   # no key: value_mask already holds the mask attached to value
      key_mask = ops.layer_mask(value if key is None else key, key_mask)
    if attention_mask is not None:
      attention_mask = ops.layer_mask(query, attention_mask)
    p = (self.query, self.key, self.value, self.attention_output)
    out, scores = ops.attention(query, value, key, *(w.kernel for w in p), *(w.bias for w in p), query_mask=query_mask,
                                value_mask=value_mask, key_mask=key_mask, attention_mask=attention_mask,
                                causal=bool(use_causal_mask), return_scores=bool(return_attention_scores))
    ops.attach_mask(out, query_mask)
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


class _BaseDenseAttention(torch.nn.Module):
  """tf-keras's BaseDenseAttention: `layer([query, value])` or `layer([query, value, key])` on ops.dense_attention.
  DESIGN.md §2 (A27) pins its rules."""

  def __init__(self, dropout: float = 0.0, seed=None, causal: bool = False, name=None, kwargs=None):
    super().__init__()
    cls = type(self).__name__
    for key, val in (kwargs or {}).items():   # Keras's base-layer arguments; anything else is a mistake
      if (key == "dtype" and val in (None, "float32", torch.float32)) or (key == "trainable" and val is True):
        continue
      if key in ("dtype", "trainable"):
        raise NotImplementedError(f"{cls}: {key}={val!r} is not supported")
      raise TypeError(f"{cls}: keyword argument not understood: {key!r}")
    if isinstance(dropout, bool) or not isinstance(dropout, (int, float)) or not 0 <= dropout < 1:
      raise ValueError(f"{type(self).__name__}: dropout must be a float in [0, 1), got {dropout!r}")
    self.dropout, self.seed, self.causal, self.name = float(dropout), seed, bool(causal), name
    self._key = 0
    if self.dropout > 0:
      if seed is None:       # drawn only when it is used, so a dropout-free layer leaves torch's RNG alone
        lo, hi = torch.randint(0, 2**32, (2,), dtype=torch.int64).tolist()
        self._key = lo | (hi << 32)
      else:
        self._key = int(seed) & (2**64 - 1)
    self._calls = 0
    self.built = False

  def _score_args(self):
    raise NotImplementedError

  def call(self, inputs, mask=None, training=None, return_attention_scores: bool = False,
           use_causal_mask: bool = False):
    cls = type(self).__name__
    if not isinstance(inputs, (list, tuple)) or len(inputs) not in (2, 3):
      raise ValueError(f"{cls} layer must be called on a list of inputs, namely [query, value] or [query, value, key]. "
                       f"Received: {inputs!r}")
    if mask is not None and (not isinstance(mask, (list, tuple)) or not 2 <= len(mask) <= len(inputs)):
      raise ValueError(f"{cls} layer mask must be a list of length 2, namely [query_mask, value_mask]. Received: "
                       f"{mask!r}")
    query, value = inputs[0], inputs[1]
    key = inputs[2] if len(inputs) == 3 else value
    for t, name in ((query, "query"), (value, "value"), (key, "key")):
      if not isinstance(t, torch.Tensor) or t.dim() != 3:
        raise ValueError(f"{cls}: {name} must be a 3-D tensor [batch, length, dim], got "
                         f"{tuple(t.shape) if isinstance(t, torch.Tensor) else type(t)}")
    if not self.built:
      self.build(int(query.shape[-1]), query.device)
    q_mask, v_mask = (None, None) if mask is None else (mask[0], mask[1])
    q_mask, v_mask = ops.layer_mask(query, q_mask), ops.layer_mask(value, v_mask)
    rate, call = 0.0, 0
    if self.dropout > 0 and resolve_training(training):
      rate, call = self.dropout, self._calls
      self._calls += 1
    mode, scale, cw = self._score_args()
    out, weights = ops.dense_attention(query, key, value, mode, scale, cw, query_mask=q_mask, value_mask=v_mask,
                                       causal=self.causal or bool(use_causal_mask), rate=rate, seed=self._key,
                                       call=call, return_scores=bool(return_attention_scores))
    ops.attach_mask(out, q_mask)
    return (out, weights) if return_attention_scores else out

  def forward(self, inputs, mask=None, training=None, return_attention_scores: bool = False,
              use_causal_mask: bool = False):
    return self.call(inputs, mask=mask, training=training, return_attention_scores=return_attention_scores,
                     use_causal_mask=use_causal_mask)

  @classmethod
  def from_config(cls, config: Dict[str, Any]):
    return cls(**config)


class Attention(_BaseDenseAttention):
  """`tf.keras.layers.Attention(use_scale=False, score_mode="dot", dropout=0.0, seed=None)`, Luong-style attention:
  `layer([query, value, key], mask=[query_mask, value_mask], training=None, return_attention_scores=False,
  use_causal_mask=False)` with query [B, Tq, dim], value [B, Tv, dv], key [B, Tv, dim] (key = value when omitted) ->
  [B, Tq, dv], and with `return_attention_scores` also the weights [B, Tq, Tv] value was multiplied by (after dropout),
  detached.  Scores: "dot" (q . k) * scale; "concat" concat_score_weight * sum_d tanh(scale (q_d + k_d)).  Weights,
  created on the first call: `scale` (a scalar, 1) with use_scale and `concat_score_weight` (a scalar, 1) with
  "concat".  A mask not passed is taken from the input an `Embedding(mask_zero=True)` produced; the value mask and the
  causal triangle (`use_causal_mask`, or the deprecated `causal=True`) drop scores before the softmax, the query mask
  zeroes output rows, and the output carries it.  Dropout on the weights in training only (`backend.resolve_training`),
  with Dropout's seed and call-counter rules.  dim and dv go up to 128 (ops.MHA_MAX_HEAD_DIM)."""

  def __init__(self, use_scale: bool = False, score_mode: str = "dot", dropout: float = 0.0, seed=None, causal=False,
               name=None, **kwargs):
    if score_mode not in ("dot", "concat"):
      raise ValueError(f"Invalid value for argument score_mode. Expected one of {{'dot', 'concat'}}. Received: "
                       f"score_mode={score_mode}")
    super().__init__(dropout, seed, causal, name, kwargs)
    self.use_scale, self.score_mode = bool(use_scale), score_mode

  def build(self, dim: int, device):
    one = lambda: torch.nn.Parameter(torch.ones((), dtype=torch.float32, device=device))
    self.scale = one() if self.use_scale else None
    self.concat_score_weight = one() if self.score_mode == "concat" else None
    self.built = True

  def _score_args(self):
    return self.score_mode, self.scale, self.concat_score_weight

  def get_config(self) -> Dict[str, Any]:
    return {"use_scale": self.use_scale, "score_mode": self.score_mode, "dropout": self.dropout, "seed": self.seed,
            "causal": self.causal, "name": self.name}


class AdditiveAttention(_BaseDenseAttention):
  """`tf.keras.layers.AdditiveAttention(use_scale=True, dropout=0.0, seed=None)`, Bahdanau-style attention: scores
  sum_d scale_d tanh(q_d + k_d), with `scale` [dim] (glorot_uniform with Keras's fans, created on the first call) when
  use_scale, else sum_d tanh(q_d + k_d).  Call, masks, dropout and the returned weights as `Attention`."""

  def __init__(self, use_scale: bool = True, dropout: float = 0.0, seed=None, causal=False, name=None, **kwargs):
    super().__init__(dropout, seed, causal, name, kwargs)
    self.use_scale = bool(use_scale)

  def build(self, dim: int, device):
    self.scale = torch.nn.Parameter(_kernel_init("glorot_uniform", (dim,), device)) if self.use_scale else None
    self.built = True

  def _score_args(self):
    return "additive", self.scale, None

  def get_config(self) -> Dict[str, Any]:
    return {"use_scale": self.use_scale, "dropout": self.dropout, "seed": self.seed, "causal": self.causal,
            "name": self.name}
