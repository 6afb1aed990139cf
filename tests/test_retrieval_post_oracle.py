"""CPU tests of tests/retrieval_post_oracle.py: the replays of the exclusion re-rank, the in-top-K count, the hit sums and
the hard-negative loss agree with the reference restatements in oracle/oracle.py, and the float64 Retrieval oracle breaks
hard-negative score ties the way tf.math.top_k does.  The GPU kernels are held to these replays in
test_gpu_retrieval_post_edges.py."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import retrieval_post_oracle as rpo  # noqa: E402
from oracle import oracle as orc  # noqa: E402

F32 = np.float32


def _int_embeddings(n, d, seed):
  """Entries in {-1, 0, 1}: every dot product is a small integer, exact in float32 and float64, so scores tie often and
  the ties are the same in both precisions."""
  return np.random.RandomState(seed).randint(-1, 2, size=(n, d)).astype(F32)


def _canonical_pos(q, c):
  return np.array([orc.scores(q[i:i + 1], c[i:i + 1])[0, 0] for i in range(q.shape[0])], F32)


# ------------------------------------------------------------------------------------------------
# exclusion re-rank
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("ties", [False, True])
def test_exclude_replay_matches_oracle_exclude(ties):
  rs = np.random.RandomState(1 + ties)
  Q, kf, E = 40, 77, 9
  if ties:   # few distinct values, +-0.0, and scores 2^-10 apart that meet after - 1e5 (ulp(1e5) = 2^-7)
    s = (F32(1.0) + rs.randint(0, 40, size=(Q, kf)).astype(F32) * F32(2.0 ** -10))
    s[:, ::5] = F32(0.0); s[:, 1::5] = F32(-0.0)
  else:
    s = rs.permutation(Q * kf).reshape(Q, kf).astype(F32) * F32(0.37) - F32(500.0)
  s = -np.sort(-s, 1)
  ids = np.stack([rs.permutation(1 << 16)[:kf] for _ in range(Q)]).astype(np.int64) << 24   # distinct, above 2^32
  ex = rs.randint(0, 1 << 16, size=(Q, E)).astype(np.int64) << 24
  ex[:, :4] = np.take_along_axis(ids, rs.randint(0, kf, size=(Q, 4)), 1)
  for k in (1, 30, kf):
    es, ei = orc.exclude(s, ids, ex, k)
    gs, gi = rpo.exclude_rerank(s, ids, ex, k)
    np.testing.assert_array_equal(gi, ei)
    np.testing.assert_array_equal(gs.view(np.uint32), es.view(np.uint32))


def test_exclude_replay_rules():
  s = np.array([[3.0, -0.0, 0.0, 2.0, 1.0, 1.0 + 2 ** -10]], F32)
  ids = np.array([[10, 11, 12, 13, 14, 15]], np.int64)
  # nothing excluded: -0.0 and +0.0 tie, so the lower position goes first
  _, i = rpo.exclude_rerank(s, ids, np.zeros((1, 0), np.int64), 6)
  assert i.tolist() == [[10, 13, 15, 14, 11, 12]]
  # 14 and 15 are excluded; 1 - 1e5 and (1 + 2^-10) - 1e5 round to the same float32, so position decides
  assert s[0, 4] - F32(1e5) == s[0, 5] - F32(1e5)
  gs, i = rpo.exclude_rerank(s, ids, np.array([[15, 14, 15, 99]], np.int64), 6)
  assert i.tolist() == [[10, 13, 11, 12, 14, 15]]
  assert gs.view(np.uint32).tolist() == [s[0, [0, 3, 1, 2, 4, 5]].view(np.uint32).tolist()]   # original scores
  # identifiers: both 13 and 14 map to identifier 7
  ident = np.zeros(20, np.int64); ident[13] = ident[14] = 7; ident[10] = 1
  _, i = rpo.exclude_rerank(s, ids, np.array([[7]], np.int64), 3, identifiers=ident)
  assert i.tolist() == [[10, 15, 11]]


# ------------------------------------------------------------------------------------------------
# in-top-K count and hit sums
# ------------------------------------------------------------------------------------------------
def test_count_and_hits_replay_match_factorized_top_k_update():
  rs = np.random.RandomState(3)
  N, d, Q, ks = 900, 16, 300, (1, 5, 10, 50)
  c = _int_embeddings(N, d, 4)
  q = _int_embeddings(Q, d, 5)
  true = c[rs.randint(0, N, Q)]
  w = rs.randint(0, 9, Q).astype(F32) * F32(0.25)   # quarter weights: every sum below is exact in float32 and float64
  exp = orc.factorized_top_k_update(q, true, lambda qq, k: orc.topk_scan(qq, c, k), ks, sample_weight=w)
  top_s, _ = orc.topk_scan(q, c, max(ks))
  pos = _canonical_pos(q, true)
  acc = rpo.hits_accumulate(rpo.count_above(top_s, pos), pos, w, ks)
  assert [a for a in acc[:-1]] == [e[0] for e in exp]
  assert acc[-1] == exp[0][1]


def test_count_above_replay_is_in_top_k():
  rs = np.random.RandomState(6)
  s = rs.randint(-3, 4, size=(64, 33)).astype(F32)
  s[3, 5:] = np.nan
  pos = rs.randint(-3, 4, size=64).astype(F32)
  pos[:3] = [np.inf, -np.inf, np.nan]
  cnt = rpo.count_above(s, pos)
  assert cnt[0] == 0 and cnt[1] == 33 and cnt[2] == 0 and cnt[3] <= 5
  for k in (1, 4, 33, 34):
    hit = orc.in_top_k(np.zeros(64, np.int64), np.concatenate([pos[:, None], s], 1), k)
    np.testing.assert_array_equal(hit, np.isfinite(pos) & (cnt < k))


def test_hits_replay_follows_the_kernel_order():
  """The vectorised replay equals a literal loop of the kernel's per-thread sums and tree, bit for bit."""
  rs = np.random.RandomState(7)
  Q, ks = 1337, (3, 1, 3)
  cnt = rs.randint(0, 5, Q).astype(np.int32)
  pos = rs.normal(size=Q).astype(F32); pos[::97] = np.inf
  w = rs.normal(size=Q).astype(F32) * F32(1e3)
  acc0 = np.array([0.5, -1.0, 3.0, 1e-3])
  got = rpo.hits_accumulate(cnt, pos, w, ks, acc0)
  for j in range(len(ks) + 1):
    red = []
    for t in range(256):
      a = 0.0
      for i in range(t, Q, 256):
        if j == len(ks) or (cnt[i] < ks[j] and np.isfinite(pos[i])):
          a += float(w[i])
      red.append(a)
    o = 128
    while o:
      for t in range(o):
        red[t] += red[t + o]
      o >>= 1
    assert got[j] == acc0[j] + red[0], j


# ------------------------------------------------------------------------------------------------
# hard-negative loss
# ------------------------------------------------------------------------------------------------
def _hardneg_replay(q, c, n, w, temp):
  """The kernels' pipeline on the CPU: the exact top-k1 list, the drop rule, float64 coefficients and gradients."""
  k1 = min(n + 1, c.shape[0])
  top_s, top_i = orc.topk_scan(q, c, k1)
  inv_t = 1.0 if temp is None else 1.0 / temp
  coef = rpo.hardneg_coefficients(top_s, top_i, _canonical_pos(q, c[:q.shape[0]]), inv_t, w)
  dq, dc, _, _ = rpo.hardneg_grads(q, c, top_i, coef)
  return coef[:, -1].sum(), dq, dc


def _close(got, ref, rel):
  ref = np.asarray(ref, np.float64)
  assert np.abs(np.asarray(got, np.float64) - ref).max() <= rel * max(np.abs(ref).max(), 1e-300)


@pytest.mark.parametrize("data", ["normal", "integer"])
@pytest.mark.parametrize("B,C,n,temp,weighted", [(37, 37, 5, None, False), (64, 200, 31, 0.05, True),
                                                  (50, 90, 40, 20.0, True), (9, 9, 100, None, True)])
def test_hardneg_replay_matches_retrieval_oracle(data, B, C, n, temp, weighted):
  rs = np.random.RandomState(B + C)
  d = 12
  if data == "normal":
    q = rs.normal(size=(B, d)).astype(F32); c = rs.normal(size=(C, d)).astype(F32)
  else:
    q = _int_embeddings(B, d, B); c = _int_embeddings(C, d, C)
  w = (rs.rand(B).astype(F32) + F32(0.25)) if weighted else None
  loss, dq, dc = _hardneg_replay(q, c, n, w, temp)
  rl, rdq, rdc = orc.retrieval_loss_and_grads_general(q, c, w, temp, num_hard_negatives=n)
  # integer scores are exact in float32: only the float32 1/T of the kernels is left
  rel = 1e-5 if data == "normal" else (1e-12 if temp is None else 1e-6)
  _close(loss, rl, rel); _close(dq, rdq, rel); _close(dc, rdc, rel)


def _tf_hard_negative_loss_and_grads(q, c, n, w, temp):
  """The reference's float32 op sequence for the selection (retrieval.py:178-208, loss.py:61-111): logits / T,
  top_k(logits + labels * MAX_FLOAT, n + 1) with tf.math.top_k's order (value desc, lower index first); then the float64
  softmax cross-entropy and its gradient over the selected columns."""
  B, C = q.shape[0], c.shape[0]
  s32 = orc.scores(q, c)
  labels = np.eye(B, C, dtype=F32)
  if temp is not None:
    s32 = s32 / F32(temp)
  _, cols = orc.top_k_rows(s32 + labels * orc.MAX_FLOAT, min(n + 1, C))
  active = np.zeros((B, C), bool)
  np.put_along_axis(active, cols, True, 1)
  t = 1.0 if temp is None else float(temp)
  s = (q.astype(np.float64) @ c.astype(np.float64).T) / t
  sm = np.where(active, s, -np.inf)
  m = sm.max(1, keepdims=True)
  e = np.exp(sm - m)
  z = e.sum(1, keepdims=True)
  w64 = np.ones(B) if w is None else w.astype(np.float64)
  eye = np.eye(B, C)
  loss = float((w64 * (m[:, 0] - (eye * s).sum(1) + np.log(z[:, 0]))).sum())
  g = (e / z - eye) * active * (w64[:, None] / t)
  return loss, g @ c.astype(np.float64), g.T @ q.astype(np.float64), cols


@pytest.mark.parametrize("temp", [None, 0.05])
def test_retrieval_oracle_breaks_hard_negative_ties_like_top_k(temp):
  """Integer embeddings with duplicated candidate rows on both sides of the positive: the float64 oracle keeps the same
  columns as tf.math.top_k on the float32 logits (lower index first among equal scores, the positive always kept)."""
  B, C, d, n = 40, 64, 6, 9
  q = _int_embeddings(B, d, 11); c = _int_embeddings(C, d, 12)
  for i in range(0, B, 3):          # a copy of the positive below it and one above it
    c[(i + 17) % C] = c[i]
    if i >= 2:
      c[i - 2] = c[i]
  w = np.random.RandomState(13).rand(B).astype(F32) + F32(0.5)
  loss, dq, dc, cols = _tf_hard_negative_loss_and_grads(q, c, n, w, temp)
  # the edge is reached: some row has a score tie with its positive cut by the n + 1 boundary
  s = orc.scores(q, c)
  cut = [i for i in range(B) if (s[i] == s[i, i]).sum() > 1 and
         ((s[i] == s[i, i]) & ~np.isin(np.arange(C), cols[i])).any()]
  assert cut
  rl, rdq, rdc = orc.retrieval_loss_and_grads_general(q, c, w, temp, num_hard_negatives=n)
  rel = 1e-12
  _close(rl, loss, rel); _close(rdq, dq, rel); _close(rdc, dc, rel)
  # and the kernels' rule (drop the positive from the raw top-(n+1), else the last entry) keeps the same columns
  rloss, rdq2, rdc2 = _hardneg_replay(q, c, n, w, temp)
  rel = 1e-12 if temp is None else 1e-6
  _close(rloss, loss, rel); _close(rdq2, dq, rel); _close(rdc2, dc, rel)
