"""NumPy oracle of multi-interest (maxsim) retrieval: a [Q, H, d] query scores candidate c by its best head,
m(q, c) = max_h s_h(c), with s_h the canonical fmaf chain of `oracle.scores` (DESIGN.md, K26).

  head_max          : the maximum over heads with a strict `>` from head 0 up, so heads that tie (+0 and -0 included) keep
                      the lowest head's bits -- the rule of tfrs_rowwise_maxsim_f32 and of K26
  topk_maxsim       : the full [Q, H, N] scores, head_max, then a stable (m desc, index asc) order
  merge_head_lists  : K26's rule replayed on given per-head lists: keep each index's best entry (higher score, then lower
                      head), order the kept entries by (score desc, index asc)
  per_head_then_merge : the GPU algorithm in NumPy (per-head top-min(k, N) by `oracle.topk_scan`, then the merge), an
                      independent check of the exactness argument
  exclude / factorized_top_k_update : `oracle.exclude` and `oracle.factorized_top_k_update` on the maxsim lists."""
from __future__ import annotations

from typing import Optional, Sequence, Tuple

import numpy as np

from oracle import oracle as orc

F32 = np.float32


def planted_case(Q: int, H: int, N: int, d: int, seed: int) -> Tuple[np.ndarray, np.ndarray]:
  """([Q, H, d] queries, [N, d] corpus) of small integers, so scores tie often, with ties planted on purpose:
  duplicate corpus rows, a duplicate head (the last one copies head 0), a zero head (+0 for every candidate) and a head
  of tiny positives that scores every 7th candidate -- rows of tiny negatives -- at -0 (the product underflows).  The
  integer heads are >= 0, so they score those rows below zero and the maximum there is a zero of either sign: the zero
  and tiny heads swap places on odd queries, so either sign sits at the lower head."""
  rs = np.random.RandomState(seed)
  q = rs.randint(0, 3, size=(Q, H, d)).astype(F32)
  c = rs.randint(-2, 3, size=(N, d)).astype(F32)
  if N >= 8:
    c[N // 2] = c[1]
    c[N - 1] = c[0]
  c[::7] = -F32(1e-30) * rs.randint(1, 3, size=(len(c[::7]), d)).astype(F32)
  if H >= 2:
    q[:, H - 1] = q[:, 0]
  if H >= 4:
    for z, t, rows in ((1, 2, slice(0, None, 2)), (2, 1, slice(1, None, 2))):
      q[rows, z] = 0.0
      q[rows, t] = F32(1e-30)
  return q, c


def head_max(per_head: np.ndarray) -> np.ndarray:
  """[..., H, n] -> [..., n]: the largest value over axis -2, the lowest head's bits among heads that tie."""
  s = np.asarray(per_head, F32)
  best = s[..., 0, :].copy()
  for h in range(1, s.shape[-2]):
    take = s[..., h, :] > best
    best = np.where(take, s[..., h, :], best)
  return best


def maxsim_scores(q3, c) -> np.ndarray:
  """[Q, N] maxsim scores of [Q, H, d] queries against a [N, d] corpus."""
  q3 = np.asarray(q3, F32)
  return head_max(np.stack([orc.scores(q3[:, h, :], c) for h in range(q3.shape[1])], 1))


def topk_maxsim(q3, c, k: int) -> Tuple[np.ndarray, np.ndarray]:
  """The exact maxsim top-min(k, N): ([Q, k'] f32, [Q, k'] int64), (m desc, index asc)."""
  m = maxsim_scores(q3, c)
  s, i = orc.top_k_rows(m, min(k, m.shape[1]))
  return s, i.astype(np.int64)


def merge_head_lists(scores, idx, k: int) -> Tuple[np.ndarray, np.ndarray]:
  """K26 on [Q, H, w] per-head lists: per query, the best entry of every index (higher score; equal scores, +-0 alike,
  keep the lower head), then the first min(k, w) kept entries by (score desc, index asc)."""
  s = np.asarray(scores, F32); ix = np.asarray(idx, np.int64)
  Q, H, w = s.shape
  k_out = min(k, w)
  out_s = np.empty((Q, k_out), F32); out_i = np.empty((Q, k_out), np.int64)
  for q in range(Q):
    best = {}
    for h in range(H):
      for r in range(w):
        i = int(ix[q, h, r])
        if i not in best or s[q, h, r] > best[i]:
          best[i] = s[q, h, r]
    keys = np.array(list(best.keys()), np.int64)
    vals = np.array([best[int(i)] for i in keys], F32)
    order = np.lexsort((keys, -vals.astype(np.float64)))[:k_out]
    out_s[q], out_i[q] = vals[order], keys[order]
  return out_s, out_i


def per_head_then_merge(q3, c, k: int) -> Tuple[np.ndarray, np.ndarray]:
  """The GPU algorithm: each of the Q*H head rows' own top-w, w = min(k, N), then merge_head_lists."""
  q3 = np.asarray(q3, F32)
  Q, H, d = q3.shape
  w = min(k, np.asarray(c).shape[0])
  s, i = orc.topk_scan(q3.reshape(Q * H, d), c, w)
  return merge_head_lists(s.reshape(Q, H, w), i.reshape(Q, H, w), k)


def brute_force(q3, c, k: int, identifiers=None):
  """BruteForce.call on [Q, H, d] queries: default identifiers are the int32 row numbers."""
  s, i = topk_maxsim(q3, c, k)
  ids = np.arange(np.asarray(c).shape[0], dtype=np.int32) if identifiers is None else np.asarray(identifiers)
  return s, ids[i]


def rowwise_maxsim(q3, c) -> np.ndarray:
  """out[r] = head_max over h of the canonical dot(q3[r, h], c[r])."""
  q3 = np.asarray(q3, F32); c = np.asarray(c, F32)
  return head_max(np.stack([np.diagonal(orc.scores(q3[:, h], c)) for h in range(q3.shape[1])], 0))


def exclude(q3, c, exclusions, k: int, identifiers=None):
  """query_with_exclusions: the maxsim top-(k + E), then the reference's `_exclude` rule."""
  ex = np.asarray(exclusions)
  s, ids = brute_force(q3, c, k + ex.shape[1], identifiers)
  return orc.exclude(s, ids, ex, k)


def factorized_top_k_update(q3, c, true_emb, ks: Sequence[int], true_ids=None, sample_weight=None,
                            identifiers=None):
  """FactorizedTopK.update_state on [Q, H, d] queries: positive = rowwise_maxsim, retrieved = the maxsim top-max(ks).
  `oracle.factorized_top_k_update` scores the positive as dot(a_r, b_r); it gets a_r = [positive_r], b_r = [1], whose
  canonical dot is the positive again (up to the sign of a zero, which no comparison sees)."""
  pos = rowwise_maxsim(q3, true_emb).reshape(-1, 1)
  return orc.factorized_top_k_update(pos, np.ones_like(pos), lambda _q, k: brute_force(q3, c, k, identifiers), ks,
                                     true_ids=true_ids, sample_weight=sample_weight)
