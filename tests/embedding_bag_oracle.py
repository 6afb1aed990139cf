"""NumPy float32 restatement of TPUEmbedding's lookups (K11, DESIGN.md section 2) and of plain SGD.

Test infrastructure: the product never imports it.  Every arithmetic step is one IEEE fp32 operation on float32 arrays
(NumPy rounds each multiply, add, divide and square root; it never contracts them), in the order DESIGN.md pins:
  pooled:    acc = acc + w*e over the bag's valid values in value order from +0; D = 1 / sum w / sqrt(sum w*w) summed the
             same way; out = acc / D (no division for sum); an empty bag gives zeros
  sequence:  out[b, j] = w_j * e_j for j < min(L, bag size), zeros elsewhere
  dense:     out[i] = e_i
  backward:  pooled (g_b * w) / D_b (g_b * w for sum); sequence g_{b,j} * w (zeros past L); dense g_i
Ids outside [0, rows) are dropped with their weights and get zero rows.
"""
from __future__ import annotations

from typing import Optional, Tuple

import numpy as np

f32 = np.float32


def _bags(row_splits: np.ndarray, n: int) -> Tuple[np.ndarray, np.ndarray]:
  sp = np.asarray(row_splits, np.int64)
  s0 = np.clip(sp[:-1], 0, n)
  s1 = np.clip(np.maximum(sp[1:], s0), 0, n)
  return s0, s1


def _prepare(table, values, weights):
  table = np.asarray(table, f32)
  ids = np.asarray(values, np.int64).reshape(-1)
  w = np.ones(ids.size, f32) if weights is None else np.asarray(weights, f32).reshape(-1)
  valid = (ids >= 0) & (ids < table.shape[0])
  return table, ids, w, valid


def lookup(table, values, row_splits=None, weights=None, combiner: str = "mean",
           max_sequence_length: int = 0) -> Tuple[np.ndarray, Optional[np.ndarray]]:
  """(activations, per-bag denominators or None).  Pooled [B, dim], sequence [B, L, dim], dense values.shape + [dim]."""
  table, ids, w, valid = _prepare(table, values, weights)
  dim = table.shape[1]
  safe = np.where(valid, ids, 0)
  if row_splits is None:
    out = np.where(valid[:, None], table[safe], f32(0)).astype(f32)
    return out.reshape(*np.shape(values), dim), None
  s0, s1 = _bags(row_splits, ids.size)
  B = s0.size
  if max_sequence_length > 0:
    L = max_sequence_length
    out = np.zeros((B, L, dim), f32)
    for j in range(L):
      m = s0 + j < s1
      v = (s0 + j)[m]
      vals = (table[safe[v]] * w[v][:, None]).astype(f32)
      out[m, j] = np.where(valid[v][:, None], vals, f32(0))
    return out, None
  acc = np.zeros((B, dim), f32)
  den = np.zeros(B, f32)
  count = np.zeros(B, np.int64)
  for j in range(int((s1 - s0).max(initial=0))):
    m = (s0 + j < s1)
    m[m] = valid[(s0 + j)[m]]
    v = (s0 + j)[m]
    acc[m] = acc[m] + w[v][:, None] * table[safe[v]]
    if combiner == "mean":
      den[m] = den[m] + w[v]
    elif combiner == "sqrtn":
      den[m] = den[m] + w[v] * w[v]
    count[m] += 1
  if combiner == "sum":
    return acc, None
  if combiner == "sqrtn":
    den = np.sqrt(den).astype(f32)
  with np.errstate(divide="ignore", invalid="ignore"):
    out = np.where((count > 0)[:, None], acc / den[:, None], acc).astype(f32)
  return out, den


def lookup_bwd(table_shape, values, grad, row_splits=None, weights=None, combiner: str = "mean",
               max_sequence_length: int = 0) -> np.ndarray:
  """The gradient rows [n, dim] of the values, in value order (the rows of the backward's (ids, rows) pair)."""
  rows, dim = table_shape
  ids = np.asarray(values, np.int64).reshape(-1)
  w = np.ones(ids.size, f32) if weights is None else np.asarray(weights, f32).reshape(-1)
  valid = (ids >= 0) & (ids < rows)
  out = np.zeros((ids.size, dim), f32)
  if row_splits is None:
    g = np.asarray(grad, f32).reshape(-1, dim)
    out[valid] = g[valid]
    return out
  s0, s1 = _bags(row_splits, ids.size)
  bag = np.full(ids.size, -1, np.int64)
  for b in range(s0.size):
    bag[s0[b]:s1[b]] = b
  pos = np.arange(ids.size) - np.where(bag >= 0, s0[np.maximum(bag, 0)], 0)
  if max_sequence_length > 0:
    g = np.asarray(grad, f32).reshape(s0.size, max_sequence_length, dim)
    m = valid & (bag >= 0) & (pos < max_sequence_length)
    out[m] = g[bag[m], pos[m]] * w[m][:, None]
    return out
  g = np.asarray(grad, f32).reshape(s0.size, dim)
  m = valid & (bag >= 0)
  r = (g[bag[m]] * w[m][:, None]).astype(f32)
  if combiner != "sum":
    _, den = lookup(np.zeros((rows, 1), f32), ids, row_splits, w, combiner)
    with np.errstate(divide="ignore", invalid="ignore"):
      r = (r / den[bag[m]][:, None]).astype(f32)
  out[m] = r
  return out


def sgd_sparse(table, ids, grad_rows, lr: float) -> np.ndarray:
  """table[id] -= lr * g once per occurrence, in order of occurrence; out-of-range ids skipped."""
  t = np.array(table, f32, copy=True)
  g = np.asarray(grad_rows, f32).reshape(-1, t.shape[1])
  lr = f32(lr)
  for i, r in enumerate(np.asarray(ids, np.int64).reshape(-1)):
    if 0 <= r < t.shape[0]:
      t[r] = t[r] - lr * g[i]
  return t


def sgd_dense(var, grad, lr: float) -> np.ndarray:
  return (np.asarray(var, f32) - f32(lr) * np.asarray(grad, f32)).astype(f32)
