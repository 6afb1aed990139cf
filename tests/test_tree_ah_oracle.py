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


def test_plan_mirrors_at_hand_computed_points():
  """The slice, chunk and merge-route mirrors at points worked out by hand on a 132-SM H100."""
  assert tao.slices(1, 1, 20000, 1, 132) == 64             # min(ceil(264 / 1), 78) capped at 64
  assert tao.slices(5, 1, 20000, 1, 132) == 53             # ceil(264 / 5)
  assert tao.slices(1, 5, 17000, 5, 132) == 13             # 3400 rows per leaf / 256
  assert tao.slices(1, 1, 1200, 2, 132) == 2
  assert tao.slices(1, 3, 20000, 10, 132) == 7             # test_gpu_tree_ah's sliced leaves
  assert tao.slices(300, 1, 20000, 1, 132) == 1 and tao.slices(1, 1, 100, 100, 132) == 1
  # 4096 queries x 10 probes x 2048 candidates: 10*2048*12 + 2048*12 + 2*128 + 4 + 10*12 + 10*12 + 10*24 B per query
  assert tao.query_chunk(4096, 10, 1, 16, 10, 2048, True) == (512 << 20) // 271076 == 1980
  assert tao.query_chunk(3, 10, 1, 16, 10, 2048, True) == 3
  assert tao.merge_region(64, 106, 106) == 6784 and tao.tree_merge(64, 106, 106)       # 162,816 B
  assert tao.merge_region(64, 107, 107) == 6848 and not tao.tree_merge(64, 107, 107)   # 164,352 B
  assert tao.tree_merge(4, 1706, 1706) and not tao.tree_merge(4, 1707, 1707)           # 163,776 / 163,872 B
  assert tao.tree_merge(64, 1, 1) and not tao.tree_merge(65, 1, 1)
  assert tao.merge_region(5, 10, 30) == 60                  # levels of 3 x 20, then 2 x 30 entries


def test_update_steps_keep_empty_members_and_signed_zero():
  xt = np.array([[-0.0, 1e8], [-0.0, 1.0], [2.0, -1e8], [-0.0, 0.5]], np.float32)
  cent = np.full((3, 2), 7.25, np.float32)
  got = tao.update_centroids(xt, np.array([0, 0, 2, 0]), cent)
  assert got[0].tobytes() == np.array([-0.0, np.float32((1e8 + 1.0 + 0.5) / 3)], np.float32).tobytes()
  assert got[1].tobytes() == cent[1].tobytes() and got[2].tobytes() == xt[2].tobytes()
  cb = np.full((2, 16, 2), 3.0, np.float32)
  cb[1, :, 1] = 0.0                                           # d = 3, dpb = 2: the last block's unused dim
  rt = np.array([[-0.0, -0.0, 1.0], [-0.0, -0.0, 2.0]], np.float32)
  got = tao.update_codebooks(rt, np.array([[5, 9], [5, 9]]), cb, 2)
  assert got[0, 5].tobytes() == np.array([-0.0, -0.0], np.float32).tobytes()
  assert np.array_equal(got[1, 9], [1.5, 0.0]) and np.all(np.delete(got[0], 5, 0) == 3.0)
  assert np.all(got[1, :, 1] == 0.0) and np.all(np.delete(got[1, :, 0], 9) == 3.0)


@pytest.mark.parametrize("dpb", [1, 3, 8])
def test_half_tie_queries_hit_half_integers(built, dpb):
  x = _data(400, 20, seed=dpb)
  cb = tao.build(x, num_leaves=4, training_iterations=1, dpb=dpb)["codebooks"]
  for t in (1.5, 2.5, -3.5, 126.5):
    q = tao.half_tie_query(cb, 20, dpb, t)
    assert q is not None, t
    T, s = tao.table(q[None], cb, dpb)
    assert s[0] == 1.0 and np.abs(T).max() == 127.0 and np.count_nonzero(T == np.float32(t)) >= 1
    T8, _ = tao.lut(q[None], cb, dpb)
    assert np.all(T8[T == np.float32(t)] == np.rint(t))      # half to even: 2, 2, -4, 126
  assert tao.half_tie_query(cb[:1], dpb, dpb, 1.5) is None
