"""Tasks: mirror of tensorflow_recommenders/tasks/{base,retrieval,ranking}.py."""
from __future__ import annotations

from typing import Callable, List, Optional, Sequence, Text, Union

import torch

from . import losses as tfrs_losses
from . import metrics as tfrs_metrics
from . import ops
from .layers import loss as loss_layers

MIN_FLOAT = loss_layers.MIN_FLOAT  # tasks/retrieval.py:25


class Task:
  """Task marker class (tasks/base.py:23-30)."""


def _categorical_crossentropy_sum(y_true: torch.Tensor, y_pred: torch.Tensor, sample_weight=None) -> torch.Tensor:
  """CategoricalCrossentropy(from_logits=True, reduction=SUM) -- the default loss, retrieval.py:86-87."""
  per = -(y_true * torch.log_softmax(y_pred, dim=1)).sum(1)
  if sample_weight is not None:
    per = per * torch.as_tensor(sample_weight, dtype=per.dtype, device=per.device).reshape(-1)
  return per.sum()


class Retrieval(torch.nn.Module, Task):
  """A factorized retrieval task (tasks/retrieval.py:29-235).

  2-D queries with the default loss run fused and never materialise the [B, C] logits or the eye() labels:
  `temperature`, the sampling-probability correction, accidental-hit removal and `score_mask` are folded into the
  tensor-core loss kernels, hard-negative mining runs on the top-K scan.  A custom loss object, multi-head (3-D)
  queries, batch metrics, or shapes outside the tensor-core range use the exact score matrix + the reference's
  op sequence."""

  def __init__(self, loss: Optional[Callable] = None,
               metrics: Optional[Union[Sequence[tfrs_metrics.Factorized], tfrs_metrics.Factorized]] = None,
               batch_metrics: Optional[List] = None, loss_metrics: Optional[List] = None,
               temperature: Optional[float] = None, num_hard_negatives: Optional[int] = None,
               remove_accidental_hits: bool = False, name: Optional[Text] = None) -> None:
    super().__init__()
    self.name = name
    self._loss = loss
    if metrics is None:
      metrics = []
    if not isinstance(metrics, Sequence):
      metrics = [metrics]
    self._factorized_metrics = list(metrics)
    self._batch_metrics = batch_metrics or []
    self._loss_metrics = loss_metrics or []
    self._temperature = temperature
    self._num_hard_negatives = num_hard_negatives
    self._remove_accidental_hits = remove_accidental_hits

  @property
  def factorized_metrics(self):
    """The metrics object used to compute retrieval metrics (:101-106)."""
    return self._factorized_metrics

  @factorized_metrics.setter
  def factorized_metrics(self, value) -> None:
    if not isinstance(value, Sequence):
      value = []
    self._factorized_metrics = list(value)

  @property
  def metrics(self):
    """Flat list of metric objects, Keras `layer.metrics` order: factorized, batch, loss metrics."""
    out = []
    for m in self._factorized_metrics:
      out.extend(m.metrics)
    return out + list(self._batch_metrics) + list(self._loss_metrics)

  def call(self, query_embeddings: torch.Tensor, candidate_embeddings: torch.Tensor,
           sample_weight: Optional[torch.Tensor] = None, candidate_sampling_probability: Optional[torch.Tensor] = None,
           candidate_ids=None, compute_metrics: bool = True, compute_batch_metrics: bool = True,
           score_mask: Optional[torch.Tensor] = None) -> torch.Tensor:
    three_d = query_embeddings.dim() == 3
    if self._remove_accidental_hits and candidate_ids is None:
      raise ValueError("When accidental hit removal is enabled, candidate ids must be supplied.")
    wants_batch_scores = compute_batch_metrics and len(self._batch_metrics) > 0
    options = (candidate_sampling_probability is not None or self._remove_accidental_hits or score_mask is not None)
    # Everything except a custom loss object, 3-D (multi-head) queries and batch metrics (which need the logits) runs
    # fused: temperature, sampling-probability correction (a per-candidate bias), accidental-hit removal (candidate ids
    # compared in the epilogue) and score_mask (keep-bits) inside the tensor-core loss; hard-negative mining through the
    # top-K scan + a sparse loss (`ops.hard_negative_softmax_loss`).  Nothing of size [B, C] is materialised there.
    fusable = not three_d and self._loss is None and not wants_batch_scores
    B_, C_, d_ = query_embeddings.shape[0], candidate_embeddings.shape[0], query_embeddings.shape[-1]
    fused_hard = (fusable and self._num_hard_negatives is not None and not options and
                  (self._temperature is None or self._temperature > 0) and
                  ops.hard_negative_supported(B_, C_, d_, self._num_hard_negatives))
    fused_opts = (fusable and self._num_hard_negatives is None and options and
                  (self._temperature is None or self._temperature > 0) and
                  ops.inbatch_softmax_bias_supported(B_, C_, d_))
    plain = not three_d and self._loss is None and self._num_hard_negatives is None and not options
    # multi-head queries (maxsim, :172-176) with the default loss: the head maximum is folded inside the blocked loss kernels.
    # Every other 3-D case takes the maximum over the head rows of the score matrix with `amax`, whose gradient -- like
    # tf.reduce_max's and the kernels' -- is split evenly among the heads that tie for the maximum.
    fused_maxsim = (three_d and self._loss is None and self._num_hard_negatives is None and not options and
                    (self._temperature is None or self._temperature > 0))
    need_scores = wants_batch_scores or not (fused_hard or fused_opts or plain or fused_maxsim)

    scores = labels = None
    if need_scores:
      if three_d:  # maxsim over query heads, :172-176
        nq, nh, e = query_embeddings.shape
        s = ops.scores(query_embeddings.reshape(nq * nh, e), candidate_embeddings)
        scores = s.reshape(nq, nh, -1).amax(dim=1)   # a tie splits the gradient evenly among the heads
      else:
        scores = ops.scores(query_embeddings, candidate_embeddings)  # :178-180
      num_queries, num_candidates = scores.shape
      labels = torch.eye(num_queries, num_candidates, device=scores.device)  # :185
      if self._temperature is not None:
        scores = scores / self._temperature
      if candidate_sampling_probability is not None:
        scores = loss_layers.SamplingProbablityCorrection()(scores, candidate_sampling_probability)
      if self._remove_accidental_hits:
        scores = loss_layers.RemoveAccidentalHits()(labels, scores, candidate_ids)
      if score_mask is not None:
        scores = torch.where(score_mask.to(scores.device).bool(), scores, torch.full_like(scores, MIN_FLOAT))
      if self._num_hard_negatives is not None:
        scores, labels = loss_layers.HardNegativeMining(self._num_hard_negatives)(scores, labels)

    if fused_opts:
      bias = None
      if candidate_sampling_probability is not None:
        # logits - log(clip(p, 1e-6, 1))  (layers/loss.py:150-158) as a bias vector
        p_c = torch.as_tensor(candidate_sampling_probability, dtype=torch.float32, device=candidate_embeddings.device).reshape(-1)
        bias = -torch.log(torch.clamp(p_c, 1e-6, 1.0))
      loss = ops.inbatch_softmax_loss(query_embeddings, candidate_embeddings, sample_weight, self._temperature, bias,
                                      candidate_ids if self._remove_accidental_hits else None,
                                      None if score_mask is None else score_mask.to(candidate_embeddings.device))
    elif fused_hard:
      loss = ops.hard_negative_softmax_loss(query_embeddings, candidate_embeddings, self._num_hard_negatives, sample_weight,
                                            self._temperature)
    elif fused_maxsim:
      loss = ops.inbatch_softmax_maxsim_loss(query_embeddings, candidate_embeddings, sample_weight, self._temperature)
    elif plain:
      loss = ops.inbatch_softmax_loss(query_embeddings, candidate_embeddings, sample_weight, self._temperature)
    elif self._loss is not None:
      loss = self._loss(labels, scores, sample_weight) if sample_weight is not None else self._loss(labels, scores)
    else:
      loss = _categorical_crossentropy_sum(labels, scores, sample_weight)

    with torch.no_grad():
      for metric in self._loss_metrics:
        metric.update_state(loss.detach())
      if compute_metrics and not three_d:
        for metric in self._factorized_metrics:
          metric.update_state(query_embeddings.detach(),
                              candidate_embeddings[:query_embeddings.shape[0]].detach(),  # :221-223
                              true_candidate_ids=candidate_ids, sample_weight=sample_weight)
      if compute_batch_metrics:
        for metric in self._batch_metrics:
          metric.update_state(labels, scores.detach(), sample_weight=sample_weight)
    return loss

  def forward(self, *args, **kwargs):
    return self.call(*args, **kwargs)


class Ranking(torch.nn.Module, Task):
  """A ranking task (tasks/ranking.py:26-119): loss of the predictions + ranking / prediction / label / loss metrics.

  A loss object of this package (`losses.BinaryCrossentropy` -- the default -- or `losses.MeanSquaredError`) runs in the
  fused ranking-loss kernel, and that same launch produces the batch statistics of every package metric of the call
  (BinaryAccuracy, AUC, (Root)MeanSquaredError, and `Mean` as a prediction / label metric); the metrics add them into their
  device-resident sums.  A listwise loss (`losses.ListMLELoss`, `PairwiseHingeLoss`, `SoftmaxLoss`) runs in the fused per-list
  kernel, and that launch also computes the NDCG of the call's `NDCGMetric`s that share the first one's topn.  Any other
  callable loss, or any other object with `update_state`, is called as is."""

  def __init__(self, loss: Optional[Callable] = None, metrics: Optional[List] = None, prediction_metrics: Optional[List] = None,
               label_metrics: Optional[List] = None, loss_metrics: Optional[List] = None, name: Optional[Text] = None) -> None:
    super().__init__()
    self.name = name
    self._loss = loss if loss is not None else tfrs_losses.BinaryCrossentropy()
    self._ranking_metrics = metrics or []
    self._prediction_metrics = prediction_metrics or []
    self._label_metrics = label_metrics or []
    self._loss_metrics = loss_metrics or []

  @property
  def metrics(self):
    """Keras `layer.metrics` order: ranking, prediction, label, loss metrics."""
    return list(self._ranking_metrics) + list(self._prediction_metrics) + list(self._label_metrics) + list(self._loss_metrics)

  def _stats_plan(self):
    """(threshold, num_thresholds, metrics served by one statistics launch): the first BinaryAccuracy threshold and AUC bucket
    count fix the launch; package metrics that need other values update themselves."""
    thr = T = None
    fused = []
    for m in self._ranking_metrics:
      if not isinstance(m, tfrs_metrics._RankingMetric):
        continue
      if m.threshold is not None and thr is not None and m.threshold != thr:
        continue
      if m.num_thresholds is not None and T is not None and m.num_thresholds != T:
        continue
      thr = m.threshold if m.threshold is not None else thr
      T = m.num_thresholds if m.num_thresholds is not None else T
      fused.append(m)
    means = [m for m in self._prediction_metrics + self._label_metrics if type(m) is tfrs_metrics.Mean]
    if not fused and not means:
      return None
    return (0.5 if thr is None else thr), (2 if T is None else T), fused

  def _ndcg_plan(self):
    """The NDCGMetrics that share the first one's topn: a listwise loss's launch computes their statistics."""
    ndcg = [m for m in self._ranking_metrics if isinstance(m, tfrs_metrics.NDCGMetric)]
    return [m for m in ndcg if m.topn == ndcg[0].topn]

  def call(self, labels: torch.Tensor, predictions: torch.Tensor, sample_weight: Optional[torch.Tensor] = None,
           training: bool = False, compute_metrics: bool = True) -> torch.Tensor:
    own_loss = isinstance(self._loss, tfrs_losses.Loss)
    listwise = isinstance(self._loss, tfrs_losses.ListwiseLoss)
    if not isinstance(labels, torch.Tensor):
      labels = torch.as_tensor(labels, dtype=torch.float32, device=predictions.device)
    plan = self._stats_plan() if compute_metrics else None
    stats = None
    ndcg_fused = self._ndcg_plan() if (listwise and compute_metrics) else []
    ndcg_stats = ops.ndcg_stats_buffer(predictions.device) if ndcg_fused else None
    if listwise:   # one K13 launch: the list loss and the NDCG of the metrics that share the first one's topn
      loss = self._loss._compute(labels, predictions, sample_weight, ndcg_stats, ndcg_fused[0].topn if ndcg_fused else None)
    elif own_loss:
      stats = None if plan is None else ops.ranking_stats_buffer(plan[1], predictions.device)
      loss = self._loss._compute(labels, predictions, sample_weight, stats, *(plan[:2] if plan else ()))
    else:
      loss = self._loss(labels, predictions, sample_weight=sample_weight)
    if not compute_metrics:
      return loss
    with torch.no_grad():
      if plan is not None and stats is None:
        stats = ops.ranking_metrics(predictions.detach(), labels, sample_weight, plan[0], plan[1])
      fused = set(map(id, plan[2])) if plan else set()
      fused_ndcg = set(map(id, ndcg_fused))
      for metric in self._ranking_metrics:
        if id(metric) in fused:
          metric._add(stats)
        elif id(metric) in fused_ndcg:
          metric._add(ndcg_stats)
        else:
          metric.update_state(y_true=labels, y_pred=predictions.detach(), sample_weight=sample_weight)
      for metrics, slot, values in ((self._prediction_metrics, 2, predictions), (self._label_metrics, 3, labels)):
        for metric in metrics:
          if type(metric) is tfrs_metrics.Mean:   # weighted sum and weight sum straight from the statistics
            metric._total = metric._total + stats[slot]
            metric._count = metric._count + stats[0]
          else:
            metric.update_state(values.detach(), sample_weight=sample_weight)
      for metric in self._loss_metrics:
        metric.update_state(loss.detach())  # a scalar that is already the weighted loss
    return loss

  def forward(self, *args, **kwargs):
    return self.call(*args, **kwargs)
