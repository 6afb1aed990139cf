"""CPU tests of the tree-AH oracle (tests/tree_ah_oracle.py) and of TreeAH's constructor checks, which run before any
kernel.  The GPU index and search are held to this oracle bit for bit in test_gpu_tree_ah.py."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import tree_ah_oracle as tao  # noqa: E402
from oracle import oracle as orc  # noqa: E402


def _data(N=3000, d=24, seed=0):
  return np.random.RandomState(seed).normal(size=(N, d)).astype(np.float32)


@pytest.fixture(scope="module")
def built():
  x = _data()
  return x, tao.build(x, num_leaves=20, training_iterations=4, dpb=4)


def test_one_leaf_full_reorder_is_brute_force():
  x = _data(500, 16)
  q = _data(7, 16, seed=1)
  idx = tao.build(x, num_leaves=1, training_iterations=2, dpb=2)
  s, i = tao.search(idx, x, q, k=10, num_leaves_to_search=1, dpb=2, num_reordering_candidates=500)
  es, ei = orc.brute_force(q, x, k=10)
  assert np.array_equal(i, ei) and np.array_equal(s, es)


def test_training_rows_sit_in_their_argmax_leaf(built):
  x, idx = built
  xt = x[idx["train_rows"]]
  d2 = ((xt[:, None, :].astype(np.float64) - idx["centroids"][None].astype(np.float64)) ** 2).sum(-1)
  leaf = idx["leaf"][idx["train_rows"]]
  # the assignment is the exact argmax of the fp32 augmented dot; in float64 it is the nearest centroid up to rounding
  assert np.all(d2[np.arange(len(leaf)), leaf] <= d2.min(1) * (1 + 1e-4) + 1e-4)
  exact = tao._aug_argmax(xt, idx["centroids"])
  assert np.array_equal(exact, leaf)


def test_centroids_are_ordered_means(built):
  x, idx = built
  # the leaf-major layout: offsets partition the rows, each leaf's rows ascending
  off, order = idx["leaf_offsets"], idx["order"]
  assert off[0] == 0 and off[-1] == x.shape[0] and np.all(np.diff(off) >= 0)
  for l in range(len(off) - 1):
    rows = order[off[l]:off[l + 1]]
    assert np.all(np.diff(rows) > 0) and np.all(idx["leaf"][rows] == l)
  # the last Lloyd step: every centroid is the ordered mean of the members the previous centroids gave it
  prev = tao.build(x, num_leaves=20, training_iterations=3, dpb=4)["centroids"]
  xt = x[idx["train_rows"]]
  a = tao._aug_argmax(xt, prev)
  for l in range(len(prev)):
    m = np.nonzero(a == l)[0]
    want = tao._ordered_mean(xt[m]) if m.size else prev[l]
    assert want.tobytes() == idx["centroids"][l].tobytes()


def test_ordered_mean_is_sequential_float64():
  rows = np.array([[1e8], [1.0], [-1e8], [0.5]], np.float32)
  assert tao._ordered_mean(rows)[0] == np.float32(((1e8 + 1.0) - 1e8 + 0.5) / 4)


def test_codes_are_nearest_centers(built):
  x, idx = built
  d, dpb = x.shape[1], 4
  B = idx["codebooks"].shape[0]
  codes = tao.unpack(idx["codes"], B)
  r = (x - idx["centroids"][idx["leaf"]])[idx["order"]]
  for b in range(B):
    c = idx["codebooks"][b]
    d2 = ((r[:, None, b * dpb:(b + 1) * dpb].astype(np.float64) - c[None].astype(np.float64)) ** 2).sum(-1)
    got = d2[np.arange(len(r)), codes[:, b]]
    assert np.all(got <= d2.min(1) * (1 + 1e-4) + 1e-5)
  assert np.array_equal(tao.pack(codes), idx["codes"])


def test_determinism():
  x = _data(800, 12)
  a = tao.build(x, num_leaves=10, training_iterations=3, dpb=3)
  b = tao.build(x, num_leaves=10, training_iterations=3, dpb=3)
  for key in ("centroids", "leaf_offsets", "order", "codebooks", "codes"):
    assert a[key].tobytes() == b[key].tobytes(), key


def test_nan_padding_and_zero_query():
  x = _data(200, 8)
  idx = tao.build(x, num_leaves=50, training_iterations=2, dpb=2)
  q = np.zeros((1, 8), np.float32)
  s, i = tao.search(idx, x, q, k=40, num_leaves_to_search=1, dpb=2)
  n = int(np.diff(idx["leaf_offsets"])[orc.topk_scan(q, idx["centroids"], 1)[1][0, 0]])
  assert n < 40 and np.all(np.isnan(s[0, n:])) and np.all(i[0, n:] == 0) and not np.any(np.isnan(s[0, :n]))


def test_constructor_checks():
  from recommenders_b200.layers import factorized_top_k as ftk
  ftk.TreeAH(parallelize_batch_searches=False)
  with pytest.raises(NotImplementedError):
    ftk.TreeAH(distance_measure="squared_l2")
  with pytest.raises(ValueError):
    ftk.TreeAH(distance_measure="cosine")
  for kw in ({"k": 0}, {"num_leaves": 0}, {"num_leaves_to_search": -1}, {"num_reordering_candidates": 0},
             {"dimensions_per_block": 0}, {"dimensions_per_block": 9}, {"k": 2049}, {"num_leaves_to_search": 3000},
             {"num_reordering_candidates": 5000}):
    with pytest.raises(ValueError):
      ftk.TreeAH(**kw)
  assert ftk.TreeAH().is_exact() is False
  with pytest.raises(ImportError):
    ftk.ScaNN()
