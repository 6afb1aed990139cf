"""CPU oracle of the ranking side (Dense layer, Keras ranking losses and metrics), used by the ranking tests.

TEST INFRASTRUCTURE ONLY, like oracle/: the product (recommenders_b200/) never imports it.  Every function cites the reference
file:line or the tf-keras contract it restates (paths relative to tensorflow_recommenders/).  The float64 functions are the
1e-5 parity bar; `dense_chain` is the canonical fp32 arithmetic of the repo (the sequential fmaf chain of
oracle/tfrs_oracle.c, reached through `oracle.scores`) for the exact Dense kernels.  The Keras loss epsilon, the sigmoid-logits
rule and the AUC bucket edges are tf-keras behaviours with no in-tree test ("parity unpinned", DESIGN.md section 2).
"""
from __future__ import annotations

import numpy as np

from oracle import oracle as orc

# ----------------------------------------------------------------------------------------------
# Dense layer / MLP   (tf.keras.layers.Dense inside layers/blocks.py:24-61, experimental/models/ranking.py:27-257)
# ----------------------------------------------------------------------------------------------
def _act64(z, act):
  if act == "relu":
    return np.maximum(z, 0.0)
  if act == "sigmoid":
    return 1.0 / (1.0 + np.exp(-z))
  return z


def dense(x, W, bias=None, activation=None) -> np.ndarray:
  """Dense.call: activation(matmul(x, kernel) + bias), kernel [in, out]; float64 (returns float64)."""
  z = np.asarray(x, np.float64) @ np.asarray(W, np.float64)
  if bias is not None:
    z = z + np.asarray(bias, np.float64)
  return _act64(z, activation)


def dense_grads(x, W, bias, gy, activation=None):
  """(dx, dW, db) of Dense.call for upstream gradient gy, float64: dz = gy * act'(z); dx = dz W^T; dW = x^T dz; db = colsum."""
  x64 = np.asarray(x, np.float64); W64 = np.asarray(W, np.float64)
  z = x64 @ W64 + (0.0 if bias is None else np.asarray(bias, np.float64))
  g = np.asarray(gy, np.float64)
  if activation == "relu":
    dz = g * (z > 0)
  elif activation == "sigmoid":
    s = 1.0 / (1.0 + np.exp(-z)); dz = g * s * (1.0 - s)
  else:
    dz = g
  return dz @ W64.T, x64.T @ dz, dz.sum(0)


def dense_chain(x, W, bias=None, activation=None, logits: bool = False):
  """Dense.call in the canonical fp32 arithmetic: z = the sequential fmaf chain over k from +0.0f (oracle.scores of x and
  kernel^T, tfrs_oracle.c dot_chain), then z + bias (one fp32 add), then relu (z > 0 ? z : 0) or sigmoid 1 / (1 + exp(-z))."""
  x = np.ascontiguousarray(x, np.float32); Wt = np.ascontiguousarray(np.asarray(W, np.float32).T)
  z = orc.scores(x, Wt)
  if bias is not None:
    z = (z + np.asarray(bias, np.float32)).astype(np.float32)
  if activation == "relu":
    y = np.where(z > 0, z, np.float32(0)).astype(np.float32)
  elif activation == "sigmoid":
    y = (np.float32(1) / (np.float32(1) + np.exp(-z))).astype(np.float32)
  else:
    y = z
  return (y, z) if logits else y


# ----------------------------------------------------------------------------------------------
# ranking task loss + metrics   (tasks/ranking.py:26-119 with the tf-keras losses / metrics it is given)
# ----------------------------------------------------------------------------------------------
KERAS_EPSILON = 1e-7   # tf.keras.backend.epsilon()


def binary_crossentropy(labels, predictions, from_logits: bool = False) -> np.ndarray:
  """tf.keras.backend.binary_crossentropy per example, float64: from probabilities p = clip(pred, eps, 1 - eps),
  -(y log(p + eps) + (1 - y) log(1 - p + eps)); from logits (tf.nn.sigmoid_cross_entropy_with_logits)
  max(z, 0) - z y + log1p(exp(-|z|)).  [B] or [B, 1] inputs: one example per row (the mean over a size-1 last axis)."""
  y = np.asarray(labels, np.float64).reshape(-1); x = np.asarray(predictions, np.float64).reshape(-1)
  if from_logits:
    return np.maximum(x, 0.0) - x * y + np.log1p(np.exp(-np.abs(x)))
  eps = np.float64(np.float32(KERAS_EPSILON))
  p = np.clip(x, eps, 1.0 - eps)
  return -(y * np.log(p + eps) + (1.0 - y) * np.log(1.0 - p + eps))


def squared_error(labels, predictions) -> np.ndarray:
  """tf.keras.losses.mean_squared_error per example ([B, 1] rows: mean over the size-1 last axis)."""
  d = np.asarray(predictions, np.float64).reshape(-1) - np.asarray(labels, np.float64).reshape(-1)
  return d * d


def ranking_loss(labels, predictions, sample_weight=None, loss: str = "bce", from_logits: bool = False,
                 reduction: str = "sum_over_batch_size"):
  """tf.keras Loss.__call__ (compute_weighted_loss): weighted per-example losses w_i l_i, then reduction "none" (the
  vector), "sum" or "sum_over_batch_size" (sum / B)."""
  per = binary_crossentropy(labels, predictions, from_logits) if loss == "bce" else squared_error(labels, predictions)
  if sample_weight is not None:
    w = np.asarray(sample_weight, np.float64).reshape(-1)
    per = per * (w if w.size == per.size else np.broadcast_to(w, per.shape))
  if reduction == "none":
    return per
  s = float(per.sum())
  return s if reduction == "sum" else (s / per.size if per.size else 0.0)


def _weights(sample_weight, n):
  return np.ones(n) if sample_weight is None else np.broadcast_to(np.asarray(sample_weight, np.float64).reshape(-1), (n,))


def binary_accuracy(labels, predictions, sample_weight=None, threshold: float = 0.5) -> float:
  """tf.keras.metrics.BinaryAccuracy: weighted mean of equal(y, cast(pred > threshold))."""
  y = np.asarray(labels, np.float64).reshape(-1); p = np.asarray(predictions, np.float32).reshape(-1)
  w = _weights(sample_weight, y.size)
  hit = (y == (p > np.float32(threshold)).astype(np.float64)).astype(np.float64)
  return float((w * hit).sum() / w.sum()) if w.sum() else 0.0


def weighted_mean(values, sample_weight=None) -> float:
  """tf.keras.metrics.Mean."""
  v = np.asarray(values, np.float64).reshape(-1)
  w = _weights(sample_weight, v.size)
  return float((w * v).sum() / w.sum()) if w.sum() else 0.0


def rmse(labels, predictions, sample_weight=None) -> float:
  """tf.keras.metrics.RootMeanSquaredError: sqrt(weighted mean of (pred - y)^2)."""
  return float(np.sqrt(weighted_mean(squared_error(labels, predictions), sample_weight)))


def auc_buckets(labels, predictions, sample_weight=None, num_thresholds: int = 200):
  """tf-keras AUC update for evenly spaced thresholds (metrics_utils._update_confusion_matrix_variables_optimized):
  bucket = max(ceil(pred (T - 1)) - 1, 0) in float32; per bucket the weighted labels and weighted (1 - labels)."""
  y = np.asarray(labels, np.float64).reshape(-1); p = np.asarray(predictions, np.float32).reshape(-1)
  w = _weights(sample_weight, y.size)
  b = np.maximum(np.ceil(p * np.float32(num_thresholds - 1)).astype(np.int64) - 1, 0)
  b = np.minimum(b, num_thresholds - 1)
  pos = np.bincount(b, weights=w * y, minlength=num_thresholds)
  neg = np.bincount(b, weights=w * (1.0 - y), minlength=num_thresholds)
  return pos, neg


def auc_from_buckets(pos, neg) -> float:
  """AUC.result() for curve="ROC", summation_method="interpolation": TP/FP at threshold i = sum of buckets >= i,
  sum_i (fpr_i - fpr_i+1) (tpr_i + tpr_i+1) / 2 with divide-no-nan rates."""
  tp = np.cumsum(np.asarray(pos, np.float64)[::-1])[::-1]; fp = np.cumsum(np.asarray(neg, np.float64)[::-1])[::-1]
  tpr = tp / tp[0] if tp[0] else np.zeros_like(tp)
  fpr = fp / fp[0] if fp[0] else np.zeros_like(fp)
  return float(np.sum((fpr[:-1] - fpr[1:]) * (tpr[:-1] + tpr[1:]) / 2.0))


def auc(labels, predictions, sample_weight=None, num_thresholds: int = 200) -> float:
  return auc_from_buckets(*auc_buckets(labels, predictions, sample_weight, num_thresholds))
