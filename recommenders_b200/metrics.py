"""Factorized top-K metrics: mirror of tensorflow_recommenders/metrics/factorized_top_k.py."""
from __future__ import annotations

import abc
from typing import List, Optional, Sequence, Union

import numpy as np
import torch

from . import ops
from .data import Dataset
from .layers import factorized_top_k as ftk


class Mean:
  """`tf.keras.metrics.Mean`: weighted running mean.  The running sums stay ON THE DEVICE (0-dim tensors): update_state
  enqueues a few small kernels and never synchronises; the host reads them once, in result()."""

  def __init__(self, name: str = "mean"):
    self.name = name
    self.reset_states()

  def reset_states(self) -> None:
    self._total = 0.0
    self._count = 0.0

  reset_state = reset_states

  def update_state(self, values, sample_weight=None) -> None:
    v = values.to(torch.float32) if isinstance(values, torch.Tensor) else torch.as_tensor(values, dtype=torch.float32)
    if sample_weight is None:
      self._total = self._total + v.sum(dtype=torch.float64); self._count = self._count + float(v.numel())
    else:
      w = sample_weight.to(torch.float32).to(v.device) if isinstance(sample_weight, torch.Tensor) \
          else torch.as_tensor(sample_weight, dtype=torch.float32, device=v.device)
      if w.numel() == v.numel():
        w = w.reshape(v.shape)
      elif w.dim() <= v.dim():
        w = torch.broadcast_to(w.reshape(w.shape + (1,) * (v.dim() - w.dim())), v.shape)
      self._total = self._total + (v * w).sum(dtype=torch.float64); self._count = self._count + w.sum(dtype=torch.float64)

  def result(self) -> float:
    count = float(self._count)
    return float(self._total) / count if count else 0.0


class _SharedMean(Mean):
  """One of FactorizedTopK's per-k means: a view on the metric's device accumulator (slot j = weighted hits of ks[j],
  last slot = the shared weight sum), so a whole update is ONE accumulate kernel and result() one read."""

  def __init__(self, owner: "FactorizedTopK", slot: int, name: str):
    self._owner, self._slot = owner, slot
    super().__init__(name)

  def reset_states(self) -> None:
    if self._owner._acc is not None:
      self._owner._acc[self._slot] = 0.0
      if self._slot == 0:
        self._owner._acc[-1] = 0.0
    self._owner._acc_host = None
    if self._slot == 0:
      self._owner._unsorted = None

  reset_state = reset_states

  def update_state(self, values, sample_weight=None) -> None:  # pragma: no cover - updates go through the owner
    raise RuntimeError("FactorizedTopK's means are updated by FactorizedTopK.update_state")

  def result(self) -> float:
    acc = self._owner._host_acc()
    return acc[self._slot] / acc[-1] if acc[-1] else 0.0


class TopKCategoricalAccuracy(Mean):
  """`tf.keras.metrics.TopKCategoricalAccuracy` (used as a batch metric in tasks/retrieval_test.py:44-47)."""

  def __init__(self, k: int = 5, name: str = "top_k_categorical_accuracy"):
    super().__init__(name)
    self.k = k

  def update_state(self, y_true, y_pred, sample_weight=None) -> None:
    target = y_true.argmax(dim=1)
    t = y_pred.gather(1, target[:, None])
    hit = ((y_pred > t).sum(1) < self.k).to(torch.float32)
    super().update_state(hit, sample_weight)


def in_top_k(targets: torch.Tensor, predictions: torch.Tensor, k: int) -> torch.Tensor:
  """tf.math.in_top_k: target's prediction is finite and fewer than k predictions are strictly larger."""
  t = predictions.gather(1, targets.to(torch.int64)[:, None])
  return torch.isfinite(t[:, 0]) & ((predictions > t).sum(1) < k)


class Factorized(torch.nn.Module, abc.ABC):
  """Computes metrics across top K candidates surfaced by a retrieval model (:27-49)."""

  @abc.abstractmethod
  def update_state(self, query_embeddings, true_candidate_embeddings, true_candidate_ids=None):
    raise NotImplementedError()

  @property
  def metrics(self) -> List[Mean]:
    return []

  def reset_states(self) -> None:
    for metric in self.metrics:
      metric.reset_states()

  def result(self) -> List[float]:
    return [metric.result() for metric in self.metrics]


class FactorizedTopK(Factorized):
  """Top-K categorical accuracy across the candidates surfaced by a retrieval layer (:52-194).

  Score branch (no `true_candidate_ids`): in_top_k(target = the positive) only needs  c_q = #{candidates scoring
  strictly above the positive}, clipped at max(ks).  When the layer can count inside its scan (`TopK.in_top_k_count`,
  e.g. a tensor-core `BruteForce` index: no top-K list, no sort) it does; otherwise it is counted on the retrieved list.
  Either way ONE kernel folds  w_q * [c_q < k]  for every k into a device accumulator -- update_state never
  synchronises with the host."""

  def __init__(self, candidates: Union[ftk.TopK, Dataset, list], ks: Sequence[int] = (1, 5, 10, 50, 100),
               name: str = "factorized_top_k") -> None:
    super().__init__()
    self.name = name
    if not isinstance(candidates, ftk.TopK):
      candidates = ftk.Streaming(k=max(ks)).index_from_dataset(candidates)  # :77-81
    self._ks = ks
    self._candidates = candidates
    self._acc = None          # float64 [len(ks) + 1] on the device: weighted hits per k, then the weight sum
    self._acc_host = None
    self._unsorted = None     # device flag: a retrieved list was not sorted (checked in result())
    self._top_k_metrics = [_SharedMean(self, j, name=f"{self.name}/top_{x}_categorical_accuracy") for j, x in enumerate(ks)]

  @property
  def metrics(self) -> List[Mean]:
    return self._top_k_metrics

  def reset_states(self) -> None:
    if self._acc is not None:
      self._acc.zero_()
    self._acc_host = None
    self._unsorted = None

  def _host_acc(self):
    if self._acc is None:
      return [0.0] * (len(self._ks) + 1)
    if self._acc_host is None:
      self._acc_host = [float(x) for x in self._acc.cpu()]   # the one synchronisation of an evaluation
      if self._unsorted is not None and bool(self._unsorted):
        raise AssertionError("Top-K predictions must be sorted.")
    return self._acc_host

  def _accumulator(self, device) -> torch.Tensor:
    if self._acc is None or self._acc.device != device:
      self._acc = torch.zeros(len(self._ks) + 1, dtype=torch.float64, device=device)
    self._acc_host = None
    return self._acc

  @torch.no_grad()
  def update_state(self, query_embeddings: torch.Tensor, true_candidate_embeddings: torch.Tensor,
                   true_candidate_ids=None, sample_weight=None) -> None:
    if true_candidate_ids is None and not self._candidates.is_exact():
      raise ValueError(f"The candidate generation layer ({self._candidates}) does not return "
                       "exact results. To perform evaluation using that layer, you must "
                       "supply `true_candidate_ids`, which will be checked against "
                       "the candidate ids returned from the candidate generation layer.")
    acc = self._accumulator(query_embeddings.device)
    kmax = max(self._ks)
    w = None if sample_weight is None else _flat_device(sample_weight, query_embeddings.device)

    if true_candidate_ids is None:
      # positive score with the same canonical chain as the retrieved scores (:133-134)
      positive_scores = ops.rowwise_dot(query_embeddings, true_candidate_embeddings)
      layer = self._candidates
      count = layer.in_top_k_count(query_embeddings, positive_scores, kmax)
      if count is None:
        top_k_predictions, _ = layer(query_embeddings, k=kmax)
        count = ops.count_above(top_k_predictions, positive_scores)
      ops.hits_accumulate(count, positive_scores, w, self._ks, acc)
      return

    top_k_predictions, retrieved_ids = self._candidates(query_embeddings, k=kmax)
    nan_padding = torch.isnan(top_k_predictions)
    # the reference asserts the retrieved list is sorted (:141-155); the check runs on the device and is raised by
    # result() -- no device->host round trip per update
    if top_k_predictions.shape[1] > 1:
      filled = torch.where(nan_padding, torch.full_like(top_k_predictions, torch.finfo(torch.float32).min), top_k_predictions)
      bad = ((filled[:, :-1] - filled[:, 1:]) < 0).any()
      self._unsorted = bad if self._unsorted is None else (self._unsorted | bad)
    if isinstance(retrieved_ids, torch.Tensor):
      tid = true_candidate_ids if isinstance(true_candidate_ids, torch.Tensor) else \
          torch.as_tensor(np.asarray(true_candidate_ids))
      tid = tid.to(retrieved_ids.device)
      if tid.dim() == 1:
        tid = tid[:, None]
      eq = (tid == retrieved_ids)
    else:
      tid = true_candidate_ids.cpu().numpy() if isinstance(true_candidate_ids, torch.Tensor) \
          else np.asarray(true_candidate_ids)
      if tid.ndim == 1:
        tid = tid[:, None]
      eq = torch.from_numpy(np.asarray(tid == np.asarray(retrieved_ids))).to(top_k_predictions.device)
    ids_match = (eq & ~nan_padding)
    # first matching position (or kmax): "match found within the first k" <=> position < k  (:157-180)
    pos_idx = torch.arange(ids_match.shape[1], device=ids_match.device, dtype=torch.int32)
    first = torch.where(ids_match, pos_idx, torch.full_like(pos_idx, ids_match.shape[1]).expand_as(ids_match)).amin(1)
    first = torch.where(first < ids_match.shape[1], first, torch.full_like(first, 2 ** 30)).to(torch.int32).contiguous()
    finite = torch.zeros(first.shape[0], dtype=torch.float32, device=first.device)
    ops.hits_accumulate(first, finite, w, self._ks, acc)


# ------------------------------------------------------------------------------------------------
# ranking metrics (the tf.keras metrics of tasks/ranking.py's tutorials and experimental/models/ranking.py)
# ------------------------------------------------------------------------------------------------
class _RankingMetric:
  """A metric whose state is a slice of the ranking statistics (`ops.ranking_metrics`, layout in include/tfrs_b200.h):
  a float64 device accumulator that update_state adds to without synchronising; result() reads it once.
  `tasks.Ranking` feeds every such metric of a call from the loss kernel's single launch (`_add`)."""

  threshold: Optional[float] = None        # the BinaryAccuracy threshold the statistics must use (None: any)
  num_thresholds: Optional[int] = None     # the AUC bucket count the statistics must use (None: any)

  def __init__(self, name: str):
    self.name = name
    self._acc = None
    self._host = None

  def _slots(self, num_thresholds: int) -> slice:
    raise NotImplementedError()

  def reset_states(self) -> None:
    if self._acc is not None:
      self._acc.zero_()
    self._host = None

  reset_state = reset_states

  def _add(self, stats: torch.Tensor) -> None:
    part = stats[self._slots((stats.numel() - ops.RANKING_STATS) // 2)]
    if self._acc is None or self._acc.device != stats.device or self._acc.shape != part.shape:
      self._acc = torch.zeros_like(part)
    self._acc.add_(part)
    self._host = None

  def update_state(self, y_true, y_pred, sample_weight=None) -> None:
    with torch.no_grad():
      self._add(ops.ranking_metrics(y_pred.detach(), torch.as_tensor(y_true, device=y_pred.device), sample_weight,
                                    0.5 if self.threshold is None else self.threshold,
                                    2 if self.num_thresholds is None else self.num_thresholds))

  def _values(self) -> np.ndarray:
    if self._acc is None:
      return None
    if self._host is None:
      self._host = self._acc.cpu().numpy()   # the one synchronisation
    return self._host


def _div_no_nan(a: float, b: float) -> float:
  return a / b if b else 0.0


class BinaryAccuracy(_RankingMetric):
  """tf.keras.metrics.BinaryAccuracy: weighted mean of [(y_pred > threshold) == y_true]."""

  def __init__(self, name: str = "binary_accuracy", dtype=None, threshold: float = 0.5):
    super().__init__(name)
    self.threshold = float(threshold)

  def _slots(self, T):
    return slice(0, 2)

  def result(self) -> float:
    v = self._values()
    return 0.0 if v is None else _div_no_nan(v[1], v[0])


class MeanSquaredError(_RankingMetric):
  """tf.keras.metrics.MeanSquaredError: weighted mean of (y_pred - y_true)^2."""

  def __init__(self, name: str = "mean_squared_error", dtype=None):
    super().__init__(name)

  def _slots(self, T):
    return slice(0, 5)

  def result(self) -> float:
    v = self._values()
    return 0.0 if v is None else _div_no_nan(v[4], v[0])


class RootMeanSquaredError(MeanSquaredError):
  """tf.keras.metrics.RootMeanSquaredError: sqrt of the weighted mean squared error."""

  def __init__(self, name: str = "root_mean_squared_error", dtype=None):
    super().__init__(name)

  def result(self) -> float:
    return float(np.sqrt(super().result()))


class AUC(_RankingMetric):
  """tf.keras.metrics.AUC with curve="ROC", summation_method="interpolation" and evenly spaced thresholds: every prediction
  adds its weighted label / (1 - label) to bucket max(ceil(p (T - 1)) - 1, 0); TP / FP at threshold i are the sums over
  buckets >= i; result = sum_i (fpr_i - fpr_i+1) (tpr_i + tpr_i+1) / 2 (divide-no-nan rates)."""

  def __init__(self, num_thresholds: int = 200, curve: str = "ROC", summation_method: str = "interpolation", name: Optional[str] = None,
               dtype=None, thresholds=None, multi_label: bool = False, num_labels=None, label_weights=None, from_logits: bool = False):
    if curve != "ROC" or summation_method != "interpolation" or multi_label or thresholds is not None or label_weights is not None \
        or from_logits:
      raise NotImplementedError("AUC: only curve='ROC', summation_method='interpolation', evenly spaced thresholds, "
                                "multi_label=False are implemented")
    if num_thresholds <= 1:
      raise ValueError("Argument `num_thresholds` must be an integer > 1. "
                       f"Received: num_thresholds={num_thresholds}")
    super().__init__(name if name is not None else "auc")
    self.num_thresholds = int(num_thresholds)

  def _slots(self, T):
    return slice(ops.RANKING_STATS, ops.RANKING_STATS + 2 * T)

  def bucket_counts(self):
    """(weighted positives, weighted negatives) per bucket, float64 NumPy arrays of length num_thresholds."""
    v = self._values()
    T = self.num_thresholds
    if v is None:
      return np.zeros(T), np.zeros(T)
    return v[:T], v[T:]

  def result(self) -> float:
    pos, neg = self.bucket_counts()
    tp = np.cumsum(pos[::-1])[::-1]; fp = np.cumsum(neg[::-1])[::-1]
    P, N = tp[0], fp[0]
    tpr = tp / P if P else np.zeros_like(tp)
    fpr = fp / N if N else np.zeros_like(fp)
    return float(np.sum((fpr[:-1] - fpr[1:]) * (tpr[:-1] + tpr[1:]) / 2.0))


class NDCGMetric:
  """tfr.keras.metrics.NDCGMetric on [B, L] lists: gain 2^y - 1, discount 1 / log2(rank + 1) truncated at `topn`, ranks by
  prediction descending (ties to the lower item), items with label < 0 are padding; result() = sum w NDCG / sum w over every
  update, one weight per list (a list without gain weighs the batch's mean weight).  The two sums are float64 on the device:
  update_state runs K13's metric-only launch and never synchronises; result() reads them once.  `tasks.Ranking` with a
  listwise loss feeds the metric from the loss launch (`_add`)."""

  def __init__(self, name: str = "ndcg_metric", topn: Optional[int] = None, gain_fn=None, rank_discount_fn=None, dtype=None,
               ragged: bool = False):
    if gain_fn is not None or rank_discount_fn is not None:
      raise NotImplementedError("NDCGMetric: custom gain_fn / rank_discount_fn are not supported")
    if ragged:
      raise NotImplementedError("NDCGMetric: ragged inputs are not supported")
    if topn is not None and topn < 1:
      raise ValueError(f"topn must be >= 1 or None, got {topn}")
    self.name = name
    self.topn = topn
    self._acc = None
    self._host = None

  def reset_states(self) -> None:
    if self._acc is not None:
      self._acc.zero_()
    self._host = None

  reset_state = reset_states

  def _add(self, stats: torch.Tensor) -> None:
    if self._acc is None or self._acc.device != stats.device:
      self._acc = torch.zeros_like(stats)
    self._acc.add_(stats)
    self._host = None

  def update_state(self, y_true, y_pred, sample_weight=None) -> None:
    self._add(ops.listwise_ndcg(y_pred.detach(), y_true, sample_weight, self.topn))

  def result(self) -> float:
    if self._acc is None:
      return 0.0
    if self._host is None:
      self._host = self._acc.cpu().numpy()   # the one synchronisation
    return _div_no_nan(float(self._host[0]), float(self._host[1]))


def _flat_device(w, device) -> torch.Tensor:
  t = w if isinstance(w, torch.Tensor) else torch.as_tensor(np.asarray(w))
  return t.to(device=device, dtype=torch.float32).reshape(-1)


def _flat(w):
  return w.reshape(-1) if isinstance(w, torch.Tensor) else np.asarray(w).reshape(-1)
