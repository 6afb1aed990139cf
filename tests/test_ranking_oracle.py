"""CPU tests of the ranking oracle (tests/ranking_oracle.py: Dense, ranking losses, ranking metrics): the reference's own known
answers (tasks/ranking_test.py:29-62) and hand-computed cases of the tf-keras contracts the GPU tests are checked against."""
import math
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import ranking_oracle as orc  # noqa: E402


@pytest.mark.parametrize("weighted", [False, True])
def test_reference_ranking_task_known_answers(weighted):
  """tasks/ranking_test.py:29-62: predictions [[1], [0.3]], labels [[1], [1]], BinaryCrossentropy + the four metrics."""
  pred = np.array([[1.0], [0.3]], np.float32); labels = np.array([[1.0], [1.0]], np.float32)
  w = np.array([1.0, 1.0], np.float32) if weighted else None
  expected_loss = -(math.log(1) + math.log(0.3)) / 2.0
  loss = orc.ranking_loss(labels, pred, w)
  assert loss == pytest.approx(expected_loss, rel=1e-6, abs=1e-6)
  assert orc.binary_accuracy(labels, pred, w) == 0.5
  assert orc.weighted_mean(labels, w) == 1.0
  assert orc.weighted_mean(pred, w) == pytest.approx(0.65, rel=1e-6)


def test_auc_hand_computed_cases():
  y = np.array([1, 1, 0, 0], np.float32)
  assert orc.auc(y, np.array([1.0, 0.9, 0.1, 0.0], np.float32)) == pytest.approx(1.0)       # perfect separation
  assert orc.auc(y, np.array([0.0, 0.1, 0.9, 1.0], np.float32)) == pytest.approx(0.0)       # reversed
  assert orc.auc(y, np.full(4, 0.5, np.float32)) == pytest.approx(0.5)                      # all equal
  # edges: p = 0 and p = 1 fall into buckets 0 and T - 2; one positive below one negative in the middle
  pos, neg = orc.auc_buckets(np.array([1, 0], np.float32), np.array([0.0, 1.0], np.float32), num_thresholds=200)
  assert pos[0] == 1 and neg[198] == 1 and pos.sum() == 1 and neg.sum() == 1
  assert orc.auc(np.array([1, 0, 1, 0], np.float32), np.array([0.8, 0.6, 0.4, 0.2], np.float32)) == pytest.approx(0.75)
  # no negatives: divide-no-nan rates
  assert orc.auc(np.ones(3, np.float32), np.array([0.1, 0.5, 0.9], np.float32)) == 0.0


def test_bce_from_logits_matches_probability_form_away_from_the_clip():
  rng = np.random.RandomState(0)
  z = rng.uniform(-6, 6, size=1000)
  y = (rng.rand(1000) > 0.5).astype(np.float64)
  p = 1.0 / (1.0 + np.exp(-z))
  a = orc.binary_crossentropy(y, z, from_logits=True)
  b = orc.binary_crossentropy(y, p)
  np.testing.assert_allclose(a, b, rtol=1e-5, atol=1e-5)
  # at the clip the probability form saturates (log(eps)), the logits form does not
  assert orc.binary_crossentropy([1.0], [0.0])[0] == pytest.approx(-math.log(2 * np.float32(1e-7)), rel=1e-6)
  assert orc.binary_crossentropy([1.0], [-40.0], from_logits=True)[0] == pytest.approx(40.0)


def test_reductions_with_weights():
  y = np.array([1.0, 0.0, 1.0], np.float32); p = np.array([0.8, 0.3, 0.6], np.float32); w = np.array([0.5, 2.0, 1.0])
  per = -(y * np.log(p.astype(np.float64) + 1e-7) + (1 - y) * np.log(1 - p.astype(np.float64) + 1e-7))
  np.testing.assert_allclose(orc.ranking_loss(y, p, w, reduction="none"), w * per, rtol=1e-6)
  assert orc.ranking_loss(y, p, w, reduction="sum") == pytest.approx(float((w * per).sum()), rel=1e-6)
  assert orc.ranking_loss(y, p, w) == pytest.approx(float((w * per).sum()) / 3, rel=1e-6)
  assert orc.ranking_loss(y, p, w, loss="mse") == pytest.approx(float((w * (p - y) ** 2).sum()) / 3, rel=1e-6)
  assert orc.rmse(y, p, w) == pytest.approx(math.sqrt(float((w * (p - y) ** 2).sum() / w.sum())), rel=1e-6)
  assert orc.binary_accuracy(y, p, w) == pytest.approx((0.5 + 2.0 + 1.0) / 3.5)


def test_dense_chain_is_the_fmaf_chain_and_agrees_with_float64():
  rng = np.random.RandomState(1)
  x = rng.normal(size=(7, 13)).astype(np.float32); W = rng.normal(size=(13, 5)).astype(np.float32)
  b = rng.normal(size=5).astype(np.float32)
  y, z = orc.dense_chain(x, W, b, "sigmoid", logits=True)
  # one output restated as the explicit chain: fma (exact product, one rounding) from +0.0f, then + bias
  acc = np.float32(0.0)
  for k in range(13):
    acc = np.float32(np.float64(x[2, k]) * np.float64(W[k, 3]) + np.float64(acc))   # exact product: float64 holds it
  assert np.float32(acc + b[3]) == z[2, 3]
  np.testing.assert_allclose(z, orc.dense(x, W, b), rtol=1e-5, atol=1e-5)
  np.testing.assert_allclose(y, orc.dense(x, W, b, "sigmoid"), rtol=1e-6, atol=1e-6)
  np.testing.assert_array_equal(orc.dense_chain(x, W, b, "relu"), np.where(z > 0, z, np.float32(0)))
  dx, dW, db = orc.dense_grads(x, W, b, np.ones((7, 5)), "relu")
  mask = (orc.dense(x, W, b) > 0).astype(np.float64)
  np.testing.assert_allclose(db, mask.sum(0)); np.testing.assert_allclose(dW, x.astype(np.float64).T @ mask)
