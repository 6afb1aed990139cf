"""NumPy replays of the per-query retrieval steps that run after a top-K list exists (csrc/topk_post.cu) and of the
hard-negative loss on such a list (csrc/hardneg.cu).

Each function restates the rule the kernel states, in the arithmetic it states:
  exclude_rerank        : float32 adjusted scores (one IEEE operation each), a stable (adjusted desc, position asc) sort
  count_above           : integer counts with a strict `>` (NaN compares false)
  hits_accumulate       : float64 sums in the kernel's fixed order (256 sequential per-thread sums, then a halving tree),
                          so the GPU accumulator can be compared bit for bit
  hardneg_coefficients  : the drop rule and the softmax coefficients in float64
  hardneg_grads         : dq, dc from given coefficients in float64, with the summands' magnitudes for a bound on the
                          float atomics of dc
The float64 Retrieval loss with every option lives in oracle/oracle.py (`retrieval_loss_and_grads_general`)."""
from __future__ import annotations

from typing import Optional, Sequence, Tuple

import numpy as np

F32 = np.float32
EXCLUDE_PENALTY = F32(1.0e5)   # factorized_top_k.py:104-107
HITS_THREADS = 256             # hits_accumulate_kernel's block size


def exclude_rerank(scores, idx, exclusions, k: int, identifiers=None) -> Tuple[np.ndarray, np.ndarray]:
  """`_exclude` on a fetched [Q, kf] list: adjusted = (excluded ? s - 1e5 : s) + 0 in float32 (the + 0 turns -0.0 into
  +0.0), the first min(k, kf) entries of a stable (adjusted desc, position asc) order, returned with their ORIGINAL
  scores and indices.  `identifiers` maps an index to the identifier the exclusions are compared with."""
  s = np.asarray(scores, F32)
  ix = np.asarray(idx, np.int64)
  ex = np.asarray(exclusions, np.int64).reshape(s.shape[0], -1)
  ident = ix if identifiers is None else np.asarray(identifiers, np.int64)[ix]
  isin = np.zeros(s.shape, bool)
  for x in range(ex.shape[1]):
    isin |= ident == ex[:, x:x + 1]
  adj = np.where(isin, s - EXCLUDE_PENALTY, s) + F32(0.0)
  assert adj.dtype == F32
  order = np.argsort(-adj, axis=1, kind="stable")[:, :min(k, s.shape[1])]
  return np.take_along_axis(s, order, 1), np.take_along_axis(ix, order, 1)


def count_above(scores, positive_scores) -> np.ndarray:
  """#{t : scores[q, t] > positive[q]} per query, int32 (tf.math.in_top_k's rule: a tie with the positive is a hit)."""
  s = np.asarray(scores, F32)
  p = np.asarray(positive_scores, F32).reshape(-1, 1)
  return (s > p).sum(1).astype(np.int32)


def _fixed_order_sum(v: np.ndarray) -> float:
  """hits_accumulate_kernel's order: thread t adds v[t], v[t + 256], ... from +0.0, then red[t] += red[t + o] for
  o = 128, 64, ..., 1.  np.add.accumulate is sequential; zero padding adds nothing (the partial sums start at +0.0 and so
  never become -0.0)."""
  rows = -(-v.shape[0] // HITS_THREADS)
  pad = np.zeros(rows * HITS_THREADS, np.float64)
  pad[:v.shape[0]] = v
  red = np.add.accumulate(pad.reshape(rows, HITS_THREADS), axis=0)[-1] if rows else np.zeros(HITS_THREADS)
  o = HITS_THREADS // 2
  while o:
    red[:o] = red[:o] + red[o:2 * o]
    o >>= 1
  return red[0]


def hits_accumulate(count, positive_scores, sample_weight: Optional[np.ndarray], ks: Sequence[int],
                    acc: Optional[np.ndarray] = None) -> np.ndarray:
  """acc[j] + sum_i w_i [count_i < ks[j] and positive_i finite]  (j < len(ks)),  acc[len(ks)] + sum_i w_i, in the
  kernel's float64 order.  Returns the new accumulator."""
  cnt = np.asarray(count, np.int64).reshape(-1)
  fin = np.isfinite(np.asarray(positive_scores, F32).reshape(-1))
  w = np.ones(cnt.shape[0]) if sample_weight is None else np.asarray(sample_weight, F32).reshape(-1).astype(np.float64)
  out = np.zeros(len(ks) + 1) if acc is None else np.array(acc, np.float64)
  for j in range(len(ks) + 1):
    v = w if j == len(ks) else np.where((cnt < int(ks[j])) & fin, w, 0.0)
    out[j] = out[j] + _fixed_order_sum(v)
  return out


def hardneg_drop(top_i) -> np.ndarray:
  """The list entry hardneg_fwd_kernel leaves out of each row's softmax: the positive (candidate `row`) where the list
  holds it, at its first position, else the list's last entry."""
  ti = np.asarray(top_i, np.int64)
  hit = ti == np.arange(ti.shape[0])[:, None]
  return np.where(hit.any(1), hit.argmax(1), ti.shape[1] - 1)


def hardneg_coefficients(top_s, top_i, positive_scores, inv_t: float, sample_weight=None) -> np.ndarray:
  """float64 [B, k1 + 2] in hardneg_fwd_kernel's layout: the coefficient of list entry t (w / T times its softmax
  probability, 0 for the dropped entry), the positive's (w / T (p - 1)), then the weighted row loss
  w (logsumexp - positive logit).  inv_t is taken as the float32 the kernel receives."""
  s = np.asarray(top_s, F32).astype(np.float64)
  B, k1 = s.shape
  inv = float(F32(inv_t))
  keep = np.ones((B, k1), bool)
  keep[np.arange(B), hardneg_drop(top_i)] = False
  lg = s * inv
  lp = np.asarray(positive_scores, F32).reshape(-1).astype(np.float64) * inv
  m = np.maximum(lp, np.where(keep, lg, -np.inf).max(1))
  e = np.where(keep, np.exp(lg - m[:, None]), 0.0)
  ep = np.exp(lp - m)
  z = e.sum(1) + ep
  w = np.ones(B) if sample_weight is None else np.asarray(sample_weight, F32).reshape(-1).astype(np.float64)
  coef = np.empty((B, k1 + 2))
  coef[:, :k1] = e / z[:, None] * (w * inv)[:, None]
  coef[:, k1] = (ep / z - 1.0) * w * inv
  coef[:, k1 + 1] = w * ((m - lp) + np.log(z))
  return coef


def hardneg_grads(q, c, top_i, coef, grad_loss: float = 1.0):
  """dq_i = g (sum_t coef_it c_{j_t} + coef_i,k1 c_i),  dc_j = g sum of coef_it q_i over every (i, t) naming j, in
  float64 from the given coefficients.  Also returns, per dc element, the sum of the summands' magnitudes and the number
  of summands (zero coefficients are skipped, as in the kernel): the reorderings of float atomics move an element by at
  most n * 2^-24 * sum|summand|."""
  q64 = np.asarray(q, F32).astype(np.float64)
  c64 = np.asarray(c, F32).astype(np.float64)
  ti = np.asarray(top_i, np.int64)
  B, k1 = ti.shape
  a = np.asarray(coef, np.float64)[:, :k1 + 1] * grad_loss
  cols = np.concatenate([ti, np.arange(B)[:, None]], 1)
  dq = np.einsum("bt,btd->bd", a, c64[cols])
  dc = np.zeros_like(c64)
  dc_abs = np.zeros_like(c64)
  n = np.zeros(c64.shape[0])
  np.add.at(dc, cols.reshape(-1), (a[:, :, None] * q64[:, None, :]).reshape(-1, q64.shape[1]))
  np.add.at(dc_abs, cols.reshape(-1), (np.abs(a)[:, :, None] * np.abs(q64)[:, None, :]).reshape(-1, q64.shape[1]))
  np.add.at(n, cols.reshape(-1), (a != 0).reshape(-1).astype(np.float64))
  return dq, dc, dc_abs, n
