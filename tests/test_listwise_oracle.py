"""CPU checks of the listwise oracle (tests/listwise_oracle.py): hand-computed known answers, finite differences, the
bit-exact float32 restatements against float64, ListMLE's tie order, the bars, and the host-side argument checks."""
import math

import numpy as np
import pytest

import listwise_oracle as lo
from recommenders_b200 import losses, metrics


def _one(mode, s, y, seed=0, call=0):
  l, g, T, n = lo.forward64(mode, np.asarray([s], np.float32), np.asarray([y], np.float32), seed=seed, call=call)
  return l[0], g[0]


# ---------------------------------------------------------------- known answers
def test_listmle_known_answers():
  l, g = _one(lo.LISTMLE, [0, 0], [1, 0])
  assert l == pytest.approx(math.log(2), abs=1e-15)
  np.testing.assert_allclose(g, [-0.5, 0.5], atol=1e-15)
  l, g = _one(lo.LISTMLE, [0, 5, 0], [1, -1, 0])          # padding in the middle
  assert l == pytest.approx(math.log(2), abs=1e-15)
  np.testing.assert_allclose(g, [-0.5, 0.0, 0.5], atol=1e-15)
  l, g = _one(lo.LISTMLE, [3, 1], [-1, 2])                 # one valid item
  assert l == 0.0 and np.all(g == 0)
  l, g = _one(lo.LISTMLE, [1, 2, 3], [-1, -1, -1])         # fully padded
  assert l == 0.0 and np.all(g == 0)
  # ties: y = (1, 1), s = (0, ln 3); order (0, 1) gives log 4, order (1, 0) gives log 4/3
  s = [0.0, math.log(3)]
  order = lo.listmle_order(np.float32([1, 1]), 0, 0, 0)
  l, _ = _one(lo.LISTMLE, s, [1, 1])
  want = math.log(4) if list(order) == [0, 1] else math.log(4) - math.log(3)
  assert l == pytest.approx(want, rel=1e-6)


def test_hinge_known_answers():
  l, g = _one(lo.HINGE, [1, 0, 3], [2, 1, 0])
  assert l == pytest.approx(7 / 3, abs=1e-15)
  np.testing.assert_allclose(g, [-1 / 3, -1 / 3, 2 / 3], atol=1e-15)
  l32, dl32, cnt = lo.hinge32(np.float32([[1, 0, 3]]), np.float32([[2, 1, 0]]))
  assert cnt[0] == 3 and l32[0] == np.float32(7) / np.float32(3)
  l, g = _one(lo.HINGE, [1, 2, 3, 4], [1, 1, -1, 1])         # all ties: no pair
  assert l == 0.0 and np.all(g == 0)
  l, g = _one(lo.HINGE, [1, 0], [1, 0])                      # margin exactly 0 at h = 0: relu'(0) = 0
  assert l == 0.0 and np.all(g == 0)


def test_softmax_known_answers():
  l, g = _one(lo.SOFTMAX, [0, 0], [1, 0])
  assert l == pytest.approx(math.log(2), abs=1e-15)
  np.testing.assert_allclose(g, [-0.5, 0.5], atol=1e-15)
  l, g = _one(lo.SOFTMAX, [0, 0, 7], [2, 2, -1])             # weighted by sum y = 4: 4 log 2 - 0
  assert l == pytest.approx(4 * math.log(2), abs=1e-14)
  np.testing.assert_allclose(g, [0.0, 0.0, 0.0], atol=1e-15)
  l, g = _one(lo.SOFTMAX, [1, 2], [0, 0])                    # all-zero labels contribute 0
  assert l == 0.0 and np.all(g == 0)


def test_ndcg_known_answers():
  y = np.float32([[3, 2, 0]])
  nd, idcg = lo.ndcg32(np.float32([[3, 2, 1]]), y)           # already ideal
  assert nd[0] == np.float32(1.0)
  nd, _ = lo.ndcg32(np.float32([[1, 2, 3]]), y)              # reversed
  want = (3 / math.log2(3) + 7 / 2) / (7 + 3 / math.log2(3))
  assert nd[0] == pytest.approx(want, rel=1e-6)
  nd, _ = lo.ndcg32(np.float32([[1, 2, 3]]), y, topn=1)      # the top item has gain 0
  assert nd[0] == 0.0
  nd, _ = lo.ndcg32(np.float32([[1, 2, 3]]), y, topn=2)
  assert nd[0] == pytest.approx((3 / math.log2(3)) / (7 + 3 / math.log2(3)), rel=1e-6)
  nd, idcg = lo.ndcg32(np.float32([[1, 2, 3]]), np.float32([[0, 0, -1]]))
  assert nd[0] == 0.0 and idcg[0] == 0.0
  nd, _ = lo.ndcg32(np.float32([[5, 5, 5]]), np.float32([[0, 1, 0]]))   # ties go to the lower index
  assert nd[0] == pytest.approx(1 / math.log2(3), rel=1e-6)


def test_ndcg_stats_weights_lists_without_gain_at_the_mean():
  nd = np.float32([1.0, 0.5, 0.0]); idcg = np.float32([1, 1, 0])
  st = lo.ndcg_stats(nd, idcg, np.float32([2, 4, 100]), 5)
  assert st[0] == 2 * 1.0 + 4 * 0.5 and st[1] == 2 + 4 + 3.0
  st = lo.ndcg_stats(nd, idcg, None, 5)
  assert st[1] == 3.0


# ---------------------------------------------------------------- finite differences
@pytest.mark.parametrize("mode", [lo.LISTMLE, lo.SOFTMAX, lo.HINGE])
def test_gradients_match_central_differences(mode):
  rng = np.random.default_rng(mode)
  y = np.float64([3, 1, -1, 0, 2, 1, -1, 4])
  s = rng.normal(size=8)
  order = lo.listmle_order(y.astype(np.float32), 0, 0, 0)
  f = {lo.LISTMLE: lambda v: lo.listmle64(v, y, order)[:2], lo.SOFTMAX: lambda v: lo.softmax64(v, y)[:2],
       lo.HINGE: lambda v: lo.hinge64(v, y)[:2]}[mode]
  _, g = f(s)
  h = 1e-6
  for i in range(len(s)):
    e = np.zeros_like(s); e[i] = h
    fd = (f(s + e)[0] - f(s - e)[0]) / (2 * h)
    assert fd == pytest.approx(g[i], abs=1e-6), (i, fd, g[i])


# ---------------------------------------------------------------- float32 restatements
def test_hinge32_agrees_with_float64_and_counts_pairs():
  rng = np.random.default_rng(3)
  s = rng.normal(size=(16, 33)).astype(np.float32)
  y = rng.integers(-1, 4, size=(16, 33)).astype(np.float32)
  w = rng.uniform(0.5, 2, size=16).astype(np.float32)
  l32, dl32, cnt = lo.hinge32(s, y, w)
  for b in range(16):
    l, g, c = lo.hinge64(s[b], y[b])
    assert c == cnt[b]
    assert l32[b] == pytest.approx(l, rel=1e-5)
    np.testing.assert_allclose(dl32[b], w[b] * g, rtol=1e-6, atol=0)


def test_fold_is_the_sum():
  v = np.random.default_rng(0).normal(size=9999)
  for L in (1, 5, 256, 1024):
    assert lo.fold(v, L) == pytest.approx(v.sum(), rel=1e-12)


# ---------------------------------------------------------------- ListMLE's tie order
def test_mix32_and_tie_order_are_reproducible_and_move_with_seed_and_call():
  i = np.arange(64)
  a = lo.mix32(1, 2, 3, i)
  assert np.array_equal(a, lo.mix32(1, 2, 3, i)) and a.dtype == np.uint32
  assert not np.array_equal(a, lo.mix32(2, 2, 3, i)) and not np.array_equal(a, lo.mix32(1, 3, 3, i))
  assert not np.array_equal(a, lo.mix32(1, 2, 4, i))
  assert int(lo.mix32(0, 0, 0, 0)) == 0          # f(0) = 0: the finalizer fixes zero
  assert int(lo.mix32(0, 0, 0, 1)) == int(lo.fmix32(1))
  y = np.ones(64, np.float32)
  o = lo.listmle_order(y, 7, 0, 0)
  assert np.array_equal(o, lo.listmle_order(y, 7, 0, 0))
  assert not np.array_equal(o, lo.listmle_order(y, 8, 0, 0)) and not np.array_equal(o, lo.listmle_order(y, 7, 1, 0))
  y2 = np.float32([0, 2, 1, 2, -1])                # labels descending first, padding dropped
  o2 = lo.listmle_order(y2, 0, 0, 0)
  assert set(o2[:2]) == {1, 3} and list(o2[2:]) == [2, 0]


# ---------------------------------------------------------------- the bars
@pytest.mark.parametrize("mode", [lo.LISTMLE, lo.SOFTMAX])
def test_bars_accept_the_float32_rounding_and_reject_a_planted_error(mode):
  rng = np.random.default_rng(11)
  pred = (rng.normal(size=(8, 37)) * 4).astype(np.float32)
  y = rng.integers(-1, 5, size=(8, 37)).astype(np.float32)
  w = rng.uniform(0.5, 2, size=8).astype(np.float32)
  l, g, T, n = lo.forward64(mode, pred, y, w, temperature=0.7)
  bars = lo.listmle_bars(l, g, T, n, w) if mode == lo.LISTMLE else lo.softmax_bars(l, g, T, n, y, w)
  wl = (w * l.astype(np.float32)).astype(np.float32)
  wg = (w[:, None].astype(np.float64) * g).astype(np.float32)
  assert lo.within(wl, w * l, bars[0]) and lo.within(wg, w[:, None] * g, bars[1])
  bad = wl.copy(); bad[3] = np.float32(bad[3] * (1 + 2.0 ** -18))
  assert not lo.within(bad, w * l, bars[0])
  k = np.unravel_index(np.argmax(np.abs(g)), g.shape)
  badg = wg.copy(); badg[k] = np.float32(badg[k] * (1 + 2.0 ** -18))
  assert not lo.within(badg, w[:, None] * g, bars[1])


# ---------------------------------------------------------------- host-side surface
def test_constructor_checks_and_config():
  for cls in (losses.ListMLELoss, losses.PairwiseHingeLoss, losses.SoftmaxLoss):
    with pytest.raises(NotImplementedError):
      cls(lambda_weight=object())
    with pytest.raises(NotImplementedError):
      cls(ragged=True)
    with pytest.raises(ValueError):
      cls(reduction="mean")
    cfg = cls(temperature=2.0).get_config()
    assert cfg["temperature"] == 2.0 and cfg["reduction"] == losses.Reduction.AUTO
  assert losses.ListMLELoss(seed=5).get_config()["seed"] == 5
  with pytest.raises(NotImplementedError):
    metrics.NDCGMetric(gain_fn=lambda y: y)
  with pytest.raises(NotImplementedError):
    metrics.NDCGMetric(rank_discount_fn=lambda r: r)
  with pytest.raises(NotImplementedError):
    metrics.NDCGMetric(ragged=True)
  m = metrics.NDCGMetric()
  assert m.name == "ndcg_metric" and m.result() == 0.0


def test_listmle_call_counter_advances_per_call():
  loss = losses.ListMLELoss(seed=9)
  assert [loss._key() for _ in range(3)] == [(9, 0), (9, 1), (9, 2)]
  assert losses.ListMLELoss()._key() == (0, 0)
