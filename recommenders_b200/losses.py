"""The tf.keras loss objects the ranking tutorials pass to `tasks.Ranking` (BinaryCrossentropy, MeanSquaredError), computed
by the fused ranking-loss kernel.  Predictions and labels are [B] or [B, 1]: one example per row."""
from __future__ import annotations

from typing import Optional

import torch

from . import ops


class Reduction:
  """tf.keras.losses.Reduction."""
  AUTO = "auto"
  NONE = "none"
  SUM = "sum"
  SUM_OVER_BATCH_SIZE = "sum_over_batch_size"


_REDUCTIONS = {Reduction.AUTO: ops.REDUCTION_SUM_OVER_BATCH_SIZE, Reduction.SUM_OVER_BATCH_SIZE: ops.REDUCTION_SUM_OVER_BATCH_SIZE,
               Reduction.SUM: ops.REDUCTION_SUM, Reduction.NONE: ops.REDUCTION_NONE}


class Loss:
  """Base of the fused losses: `loss(y_true, y_pred, sample_weight=None)` with the Keras reductions (AUTO =
  SUM_OVER_BATCH_SIZE: sum_i w_i l_i / B; SUM; NONE: the weighted per-example losses)."""

  def __init__(self, reduction: str = Reduction.AUTO, name: Optional[str] = None):
    if reduction not in _REDUCTIONS:
      raise ValueError(f"Invalid Reduction Key: {reduction}. Expected keys are {tuple(_REDUCTIONS)}")
    self.reduction = reduction
    self.name = name

  def _inputs(self, y_pred: torch.Tensor):
    """(tensor the loss reads, loss kind)."""
    raise NotImplementedError()

  def _compute(self, y_true, y_pred, sample_weight=None, stats=None, threshold: float = 0.5, num_thresholds: int = 200):
    loss_in, kind = self._inputs(y_pred)
    return ops.ranking_loss(loss_in, y_true, sample_weight, kind, _REDUCTIONS[self.reduction], pred=y_pred.detach(), stats=stats,
                            threshold=threshold, num_thresholds=num_thresholds)

  def __call__(self, y_true, y_pred, sample_weight=None) -> torch.Tensor:
    return self._compute(y_true, y_pred, sample_weight)

  def get_config(self):
    return {"reduction": self.reduction, "name": self.name}


class BinaryCrossentropy(Loss):
  """tf.keras.losses.BinaryCrossentropy.  from_logits=False: p = clip(y_pred, 1e-7, 1 - 1e-7),
  l = -(y log(p + 1e-7) + (1 - y) log(1 - p + 1e-7)); a prediction produced by a fused sigmoid Dense is scored from the logits
  it carries (max(z, 0) - z y + log1p(exp(-|z|))), as tf-keras does with the logits of a sigmoid output."""

  def __init__(self, from_logits: bool = False, label_smoothing: float = 0.0, axis: int = -1, reduction: str = Reduction.AUTO,
               name: str = "binary_crossentropy"):
    super().__init__(reduction, name)
    if label_smoothing:
      raise NotImplementedError("BinaryCrossentropy: label_smoothing is not supported")
    self.from_logits = from_logits
    self.label_smoothing = label_smoothing
    self.axis = axis

  def _inputs(self, y_pred):
    if self.from_logits:
      return y_pred, ops.LOSS_BCE_LOGITS
    logits = ops.attached_logits(y_pred)
    if logits is not None:
      return logits, ops.LOSS_BCE_LOGITS
    return y_pred, ops.LOSS_BCE

  def get_config(self):
    return {**super().get_config(), "from_logits": self.from_logits, "label_smoothing": self.label_smoothing, "axis": self.axis}


class MeanSquaredError(Loss):
  """tf.keras.losses.MeanSquaredError: l = (y_pred - y)^2."""

  def __init__(self, reduction: str = Reduction.AUTO, name: str = "mean_squared_error"):
    super().__init__(reduction, name)

  def _inputs(self, y_pred):
    return y_pred, ops.LOSS_MSE
