"""The loss objects the ranking tutorials pass to `tasks.Ranking`.

The tf.keras pointwise losses (BinaryCrossentropy, MeanSquaredError) run in the fused ranking-loss kernel; predictions and
labels are [B] or [B, 1], one example per row.  TF-Ranking's listwise losses (ListMLELoss, PairwiseHingeLoss, SoftmaxLoss)
run in the fused per-list kernel K13; predictions and labels are [B, L] (or [B, L, 1]), one list per row, and an item with
label < 0 is padding.  Their rules are in DESIGN.md §2 (A18)."""
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


class ListwiseLoss:
  """Base of TF-Ranking's listwise Keras losses (`tfr.keras.losses`): `loss(y_true, y_pred, sample_weight=None)` on [B, L]
  lists with one weight per list ([B] or [B, 1]) and the Keras reductions (AUTO = SUM_OVER_BATCH_SIZE: sum_b w_b l_b / B;
  SUM; NONE: the weighted per-list losses [B]).  Scores are divided by `temperature` (one fp32 multiply by 1/T)."""

  _mode = None

  def __init__(self, reduction: str = Reduction.AUTO, name: Optional[str] = None, lambda_weight=None, temperature: float = 1.0,
               ragged: bool = False):
    if reduction not in _REDUCTIONS:
      raise ValueError(f"Invalid Reduction Key: {reduction}. Expected keys are {tuple(_REDUCTIONS)}")
    if lambda_weight is not None:
      raise NotImplementedError(f"{type(self).__name__}: lambda_weight is not supported")
    if ragged:
      raise NotImplementedError(f"{type(self).__name__}: ragged inputs are not supported")
    if not temperature > 0:
      raise ValueError(f"temperature must be > 0, got {temperature}")
    self.reduction = reduction
    self.name = name
    self.lambda_weight = lambda_weight
    self.temperature = float(temperature)
    self.ragged = ragged

  def _key(self):
    """(seed, call) of ListMLE's tie order; 0 for the other losses."""
    return 0, 0

  def _compute(self, y_true, y_pred, sample_weight=None, ndcg_stats=None, topn=None) -> torch.Tensor:
    seed, call = self._key()
    return ops.listwise_loss(y_pred, y_true, sample_weight, self._mode, _REDUCTIONS[self.reduction], self.temperature, seed, call,
                             ndcg_stats, topn)

  def __call__(self, y_true, y_pred, sample_weight=None) -> torch.Tensor:
    return self._compute(y_true, y_pred, sample_weight)

  def get_config(self):
    return {"reduction": self.reduction, "name": self.name, "lambda_weight": self.lambda_weight, "temperature": self.temperature,
            "ragged": self.ragged}


class ListMLELoss(ListwiseLoss):
  """tfr.keras.losses.ListMLELoss: the negative log-likelihood of the label-sorted permutation under the Plackett-Luce model,
  l = sum_k log sum_{j >= k} exp(s_pi(j)) - s_pi(k).  Label ties are broken by a hash of (seed, call, list, item), `call` being
  this object's call counter, so every call shuffles ties differently and reproducibly."""

  _mode = ops.LIST_LOSS_LISTMLE

  def __init__(self, reduction: str = Reduction.AUTO, name: str = "list_mle_loss", lambda_weight=None, temperature: float = 1.0,
               ragged: bool = False, seed: Optional[int] = None):
    super().__init__(reduction, name, lambda_weight, temperature, ragged)
    self.seed = seed
    self._calls = 0

  def _key(self):
    call = self._calls
    self._calls += 1
    return (0 if self.seed is None else int(self.seed)), call

  def get_config(self):
    return {**super().get_config(), "seed": self.seed}


class PairwiseHingeLoss(ListwiseLoss):
  """tfr.keras.losses.PairwiseHingeLoss: the mean over the list's pairs (y_i > y_j) of max(0, 1 - (s_i - s_j))."""

  _mode = ops.LIST_LOSS_PAIRWISE_HINGE

  def __init__(self, reduction: str = Reduction.AUTO, name: str = "pairwise_hinge_loss", lambda_weight=None,
               temperature: float = 1.0, ragged: bool = False):
    super().__init__(reduction, name, lambda_weight, temperature, ragged)


class SoftmaxLoss(ListwiseLoss):
  """tfr.keras.losses.SoftmaxLoss: the cross-entropy of softmax(s) against the labels normalised to sum 1, weighted by the
  label sum: l = -sum_i y_i log_softmax(s)_i."""

  _mode = ops.LIST_LOSS_SOFTMAX

  def __init__(self, reduction: str = Reduction.AUTO, name: str = "softmax_loss", lambda_weight=None, temperature: float = 1.0,
               ragged: bool = False):
    super().__init__(reduction, name, lambda_weight, temperature, ragged)
