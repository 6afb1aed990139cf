"""`LayerNormalization`, the normalization of Transformer blocks: tf.keras.layers.LayerNormalization over the last axis
on K22.  DESIGN.md §2 (A25) pins its rule.  `BatchNormalization`, the normalization of MLP towers, on K24 (A26)."""
from __future__ import annotations

from typing import Any, Dict

import torch

from .. import ops
from ..backend import resolve_training
from .feature_interaction.dcn import _init


class LayerNormalization(torch.nn.Module):
  """`tf.keras.layers.LayerNormalization()`: y = (x - mean) * rsqrt(var + epsilon) * gamma + beta over the last axis of x
  (float32), with the population variance.  gamma [d] ("ones") and beta [d] ("zeros") are created on the first call;
  `scale=False` / `center=False` leave them out.  A mask attached to x (an `Embedding(mask_zero=True)` output) is
  attached to y too.  Any axis but the last, regularizers and constraints raise NotImplementedError."""

  def __init__(self, axis=-1, epsilon: float = 1e-3, center: bool = True, scale: bool = True,
               beta_initializer="zeros", gamma_initializer="ones", beta_regularizer=None, gamma_regularizer=None,
               beta_constraint=None, gamma_constraint=None, name=None, **kwargs):
    super().__init__()
    unsupported = {
        "beta_regularizer": beta_regularizer is not None,
        "gamma_regularizer": gamma_regularizer is not None,
        "beta_constraint": beta_constraint is not None,
        "gamma_constraint": gamma_constraint is not None,
    }
    for arg, bad in unsupported.items():
      if bad:
        raise NotImplementedError(f"LayerNormalization: {arg}={locals()[arg]!r} is not supported")
    self.axis = list(axis) if isinstance(axis, (list, tuple)) else axis
    if isinstance(self.axis, list) and len(self.axis) != 1:
      raise NotImplementedError(f"LayerNormalization: axis={axis!r} is not supported (the last axis only)")
    self.epsilon, self.center, self.scale = float(epsilon), bool(center), bool(scale)
    self._beta_initializer, self._gamma_initializer = beta_initializer, gamma_initializer
    self.name = name
    self.built = False

  def _check_axis(self, rank: int) -> None:
    a = self.axis[0] if isinstance(self.axis, list) else self.axis
    if a not in (-1, rank - 1):
      raise NotImplementedError(f"LayerNormalization: axis={self.axis!r} is not supported (the last axis only)")

  def build(self, input_shape, device=None):
    self._check_axis(len(input_shape))
    d = int(input_shape[-1])
    device = device or torch.device("cuda", torch.cuda.current_device())
    self.gamma = torch.nn.Parameter(_init(self._gamma_initializer, (d,), device)) if self.scale else None
    self.beta = torch.nn.Parameter(_init(self._beta_initializer, (d,), device)) if self.center else None
    self.built = True

  def call(self, inputs: torch.Tensor, training=None):
    if not isinstance(inputs, torch.Tensor):
      raise TypeError(f"LayerNormalization: inputs must be a torch.Tensor, got {type(inputs)}")
    if not self.built:
      self.build(inputs.shape, inputs.device)
    self._check_axis(inputs.dim())
    mask = ops.attached_mask(inputs)
    return ops.attach_mask(ops.layer_norm(inputs, self.gamma, self.beta, self.epsilon), mask)

  def forward(self, inputs, training=None):
    return self.call(inputs, training=training)

  def get_config(self) -> Dict[str, Any]:
    return {"axis": self.axis, "epsilon": self.epsilon, "center": self.center, "scale": self.scale,
            "beta_initializer": self._beta_initializer, "gamma_initializer": self._gamma_initializer,
            "beta_regularizer": None, "gamma_regularizer": None, "beta_constraint": None, "gamma_constraint": None,
            "name": self.name}

  @classmethod
  def from_config(cls, config: Dict[str, Any]):
    return cls(**config)


class BatchNormalization(torch.nn.Module):
  """`tf.keras.layers.BatchNormalization()` over the last axis of x (float32, rank >= 2; the statistics run over every
  other axis).  In training: y = (x - mean) * rsqrt(var + epsilon) * gamma + beta with the batch mean and population
  variance, and the moving statistics move toward them with decay 1 - momentum; at inference the moving statistics stand
  in for the batch's.  `training` resolves as `backend.resolve_training` says: the argument, then the innermost
  learning-phase scope (`Model.train_step` opens a training one), then False.

  gamma ("ones") and beta ("zeros") are Parameters created on the first call; `scale=False` / `center=False` leave them
  out.  moving_mean ("zeros") and moving_variance ("ones") are registered buffers: they are in `state_dict`, and no
  optimizer sees them.  A mask (x.shape[:-1], passed as `mask=` or attached by `Embedding(mask_zero=True)`) restricts the
  batch moments to the kept rows (tf-keras's masked weighted moments) and is attached to the output.  Any axis but the
  last, renorm, virtual_batch_size, adjustment, synchronized=True, trainable=False, regularizers and constraints raise
  NotImplementedError."""

  def __init__(self, axis=-1, momentum: float = 0.99, epsilon: float = 1e-3, center: bool = True, scale: bool = True,
               beta_initializer="zeros", gamma_initializer="ones", moving_mean_initializer="zeros",
               moving_variance_initializer="ones", beta_regularizer=None, gamma_regularizer=None, beta_constraint=None,
               gamma_constraint=None, renorm: bool = False, renorm_clipping=None, renorm_momentum: float = 0.99,
               fused=None, trainable: bool = True, virtual_batch_size=None, adjustment=None, name=None,
               synchronized: bool = False, **kwargs):
    super().__init__()
    unsupported = {
        "beta_regularizer": beta_regularizer is not None,
        "gamma_regularizer": gamma_regularizer is not None,
        "beta_constraint": beta_constraint is not None,
        "gamma_constraint": gamma_constraint is not None,
        "renorm": bool(renorm),
        "renorm_clipping": renorm_clipping is not None,
        "virtual_batch_size": virtual_batch_size is not None,
        "adjustment": adjustment is not None,
        "synchronized": bool(synchronized),
        "trainable": not trainable,
    }
    for arg, bad in unsupported.items():
      if bad:
        raise NotImplementedError(f"BatchNormalization: {arg}={locals()[arg]!r} is not supported")
    self.axis = list(axis) if isinstance(axis, (list, tuple)) else axis
    if isinstance(self.axis, list) and len(self.axis) != 1:
      raise NotImplementedError(f"BatchNormalization: axis={axis!r} is not supported (the last axis only)")
    self.momentum, self.epsilon = float(momentum), float(epsilon)
    self.center, self.scale = bool(center), bool(scale)
    self._beta_initializer, self._gamma_initializer = beta_initializer, gamma_initializer
    self._moving_mean_initializer, self._moving_variance_initializer = moving_mean_initializer, moving_variance_initializer
    self.name = name
    self.built = False

  def _check_axis(self, rank: int) -> None:
    a = self.axis[0] if isinstance(self.axis, list) else self.axis
    if a not in (-1, rank - 1):
      raise NotImplementedError(f"BatchNormalization: axis={self.axis!r} is not supported (the last axis only)")

  def build(self, input_shape, device=None):
    if len(input_shape) < 2:
      raise ValueError(f"BatchNormalization: the input must have at least two axes, got shape {tuple(input_shape)}")
    self._check_axis(len(input_shape))
    d = int(input_shape[-1])
    device = device or torch.device("cuda", torch.cuda.current_device())
    self.gamma = torch.nn.Parameter(_init(self._gamma_initializer, (d,), device)) if self.scale else None
    self.beta = torch.nn.Parameter(_init(self._beta_initializer, (d,), device)) if self.center else None
    self.register_buffer("moving_mean", _init(self._moving_mean_initializer, (d,), device))
    self.register_buffer("moving_variance", _init(self._moving_variance_initializer, (d,), device))
    self.built = True

  def call(self, inputs: torch.Tensor, training=None, mask=None):
    if not isinstance(inputs, torch.Tensor):
      raise TypeError(f"BatchNormalization: inputs must be a torch.Tensor, got {type(inputs)}")
    if not self.built:
      self.build(inputs.shape, inputs.device)
    self._check_axis(inputs.dim())
    mask = ops.layer_mask(inputs, mask)
    y = ops.batch_norm(inputs, self.gamma, self.beta, self.moving_mean, self.moving_variance,
                       resolve_training(training), self.momentum, self.epsilon, mask)
    return ops.attach_mask(y, mask)

  def forward(self, inputs, training=None, mask=None):
    return self.call(inputs, training=training, mask=mask)

  def get_config(self) -> Dict[str, Any]:
    return {"axis": self.axis, "momentum": self.momentum, "epsilon": self.epsilon, "center": self.center,
            "scale": self.scale, "beta_initializer": self._beta_initializer,
            "gamma_initializer": self._gamma_initializer, "moving_mean_initializer": self._moving_mean_initializer,
            "moving_variance_initializer": self._moving_variance_initializer, "beta_regularizer": None,
            "gamma_regularizer": None, "beta_constraint": None, "gamma_constraint": None, "name": self.name}

  @classmethod
  def from_config(cls, config: Dict[str, Any]):
    return cls(**config)
