"""GPU tests of TreeAH (K9): the reference's ScaNN tests (layers/factorized_top_k_test.py:183-258,
metrics/factorized_top_k_test.py:88-131) restated for TreeAH, and bit-exact parity of the index and the search with
tests/tree_ah_oracle.py.  Run with -m gpu."""
import itertools
import os
import sys

import numpy as np
import pytest
import torch

from oracle import oracle as orc

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import tree_ah_oracle as tao  # noqa: E402

pytestmark = pytest.mark.gpu

INDEX_KEYS = ("centroids", "leaf_offsets", "order", "codebooks", "codes")


def cu(a):
  return torch.from_numpy(np.ascontiguousarray(a)).cuda()


@pytest.fixture(scope="module")
def ftk():
  from recommenders_b200.layers import factorized_top_k
  return factorized_top_k


@pytest.fixture(scope="module")
def Dataset():
  from recommenders_b200.data import Dataset as D
  return D


def _np(t):
  return t.cpu().numpy() if isinstance(t, torch.Tensor) else np.asarray(t)


def _same(got_s, got_i, exp_s, exp_i):
  np.testing.assert_array_equal(_np(got_i), exp_i)
  assert _np(got_s).tobytes() == np.ascontiguousarray(exp_s, np.float32).tobytes()


# ---- the reference's ScaNN tests ------------------------------------------------------------------------------------
@pytest.mark.parametrize("k,batch_size,num_queries,num_candidates,indices_dtype,use_exclusions",
                         list(itertools.product((5, 10), (3, 16), (3, 15, 16), (1024, 128), (str, None), (True, False))))
def test_scann_top_k(ftk, Dataset, k, batch_size, num_queries, num_candidates, indices_dtype, use_exclusions):
  """factorized_top_k_test.py:245-258: one leaf, every row reordered -> exactly the brute force, bit for bit."""
  rng = np.random.RandomState(42)
  candidates = rng.normal(size=(num_candidates, 4)).astype(np.float32)
  query = rng.normal(size=(num_queries, 4)).astype(np.float32)
  ids = np.arange(num_candidates).astype(indices_dtype if indices_dtype is not None else np.int32)
  exclude = rng.randint(0, num_candidates, size=(num_queries, 5))
  layer = ftk.TreeAH(k=k, num_leaves=1, num_leaves_to_search=1, num_reordering_candidates=num_candidates)
  ds = Dataset.from_tensor_slices(cu(candidates)).batch(batch_size)
  if indices_dtype is not None:
    ds = Dataset.zip((Dataset.from_tensor_slices(ids).batch(batch_size), ds))
  excl = ids[exclude]
  excl_arg = excl if indices_dtype is not None else cu(excl)
  bf = lambda q, kk: orc.brute_force(q, candidates, ids, k=kk)
  exp_s, exp_i = orc.query_with_exclusions(bf, query, excl, k) if use_exclusions else bf(query, k)
  for _ in range(2):
    layer.index_from_dataset(ds)
    s, i = layer.query_with_exclusions(cu(query), excl_arg) if use_exclusions else layer(cu(query))
  _same(s, i, exp_s, exp_i)
  restored = ftk.TreeAH(k=k, num_leaves=1, num_leaves_to_search=1, num_reordering_candidates=num_candidates)
  restored.load_state_dict(layer.state_dict())
  _, ri = restored.query_with_exclusions(cu(query), excl_arg) if use_exclusions else restored(cu(query))
  np.testing.assert_array_equal(_np(ri), exp_i)


def _save_and_restore(ftk, layer, query, num=100):
  """factorized_top_k_test.py:71-83, with a state_dict round trip instead of a SavedModel."""
  first = [_np(t) for t in layer(query)]
  for _ in range(num - 1):
    again = [_np(t) for t in layer(query)]
    assert all(a.tobytes() == b.tobytes() for a, b in zip(first, again))
  restored = ftk.TreeAH()
  restored.load_state_dict(layer.state_dict())
  for _ in range(num):
    again = [_np(t) for t in restored(query)]
    assert all(np.array_equal(a, b) for a, b in zip(first, again))
  return first


@pytest.mark.parametrize("identifier_dtype", [str, np.float32, np.float64, np.int32, np.int64])
def test_scann(ftk, identifier_dtype):
  """factorized_top_k_test.py:185-198."""
  rng = np.random.RandomState(42)
  candidates = rng.normal(size=(1000, 4)).astype(np.float32)
  query = rng.normal(size=(4, 4)).astype(np.float32)
  names = np.arange(1000).astype(identifier_dtype)
  names = names if identifier_dtype is str else cu(names)
  layer = ftk.TreeAH().index(cu(candidates), names)
  s, i = _save_and_restore(ftk, layer, cu(query))
  idx = tao.build(candidates, 100, 12, 2)
  es, ei = tao.search(idx, candidates, query, 10, 10, 2)
  assert s.tobytes() == es.tobytes()
  np.testing.assert_array_equal(i, np.arange(1000).astype(identifier_dtype)[ei])


def test_scann_dataset_arg_no_identifiers(ftk, Dataset):
  """factorized_top_k_test.py:200-212."""
  rng = np.random.RandomState(42)
  candidates = rng.normal(size=(100, 4)).astype(np.float32)
  query = rng.normal(size=(4, 4)).astype(np.float32)
  layer = ftk.TreeAH().index_from_dataset(Dataset.from_tensor_slices(cu(candidates)).batch(100))
  s, i = _save_and_restore(ftk, layer, cu(query))
  es, ei = tao.search(tao.build(candidates, 100, 12, 2), candidates, query, 10, 10, 2)
  assert s.tobytes() == es.tobytes() and np.array_equal(i, ei)


def test_scann_dataset_arg_with_identifiers(ftk, Dataset):
  """factorized_top_k_test.py:214-227."""
  rng = np.random.RandomState(42)
  candidates = rng.normal(size=(100, 4)).astype(np.float32)
  query = rng.normal(size=(4, 4)).astype(np.float32)
  ids = cu(np.arange(100) + 1000)
  layer = ftk.TreeAH().index_from_dataset(Dataset.zip((Dataset.from_tensor_slices(ids).batch(100),
                                                       Dataset.from_tensor_slices(cu(candidates)).batch(100))))
  s, i = _save_and_restore(ftk, layer, cu(query))
  es, ei = tao.search(tao.build(candidates, 100, 12, 2), candidates, query, 10, 10, 2)
  assert s.tobytes() == es.tobytes() and np.array_equal(i, ei + 1000)


def test_raise_on_incorrect_input_shape(ftk, Dataset):
  """factorized_top_k_test.py:229-243, plus the rank and size checks of TreeAH."""
  cands = cu(np.random.normal(size=(100, 4)).astype(np.float32))
  with pytest.raises(ValueError):
    ftk.TreeAH().index_from_dataset(Dataset.zip((Dataset.from_tensor_slices(np.arange(99)).batch(20),
                                                 Dataset.from_tensor_slices(cands).batch(100))))
  with pytest.raises(ValueError):
    ftk.TreeAH().index(cands, np.arange(99))
  with pytest.raises(ValueError):
    ftk.TreeAH().index(cands.reshape(-1))
  with pytest.raises(ValueError):
    ftk.TreeAH().index(cu(np.zeros((10, 257), np.float32)))
  with pytest.raises(ValueError):
    ftk.TreeAH()(cands[:2])
  layer = ftk.TreeAH().index(cands)
  with pytest.raises(ValueError, match="Queries must be of rank 2 or 1"):
    layer(cands.reshape(10, 10, 4))


def test_id_based_evaluation(ftk, Dataset):
  """metrics/factorized_top_k_test.py:88-131 at default settings, one-query calls."""
  from recommenders_b200 import metrics
  rng = np.random.default_rng(42)
  k, N, Q, d = 100, 1280, 128, 128
  cand = rng.normal(size=(N, d)).astype(np.float32)
  qs = rng.normal(size=(Q, d)).astype(np.float32)
  true_idx = rng.integers(0, N, size=Q).astype(np.int32)
  index = ftk.TreeAH(k=k).index_from_dataset(Dataset.from_tensor_slices(cu(cand)).batch(32))
  metric = metrics.FactorizedTopK(candidates=index, ks=[k])
  with pytest.raises(ValueError):
    metric.update_state(cu(qs[:1]), cu(cand[:1]))
  hits = 0
  tq, tc = cu(qs), cu(cand)
  for i in range(Q):
    metric.update_state(tq[i:i + 1], tc[int(true_idx[i])].reshape(1, -1), cu(true_idx[i:i + 1]))
    _, ti = index(tq[i:i + 1])
    hits += int(int(true_idx[i]) in ti[0].cpu().tolist())
  assert metric.result()[0] == hits / Q
  es, ei = tao.search(tao.build(cand, 100, 12, 2), cand, qs, k, 10, 2)
  s, i = index(tq)
  _same(s, i, es, ei)


# ---- build parity ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("N,d,dpb,L,iters", [(20000, 64, 2, 100, 12), (20000, 42, 4, 64, 12), (150000, 32, 1, 256, 4)])
def test_build_parity(ftk, N, d, dpb, L, iters):
  x = np.random.default_rng(N + d).normal(size=(N, d)).astype(np.float32)
  layer = ftk.TreeAH(num_leaves=L, training_iterations=iters, dimensions_per_block=dpb).index(cu(x))
  exp = tao.build(x, L, iters, dpb)
  for key in INDEX_KEYS:
    got = _np(layer._index[key])
    assert got.shape == exp[key].shape, key
    assert got.tobytes() == np.ascontiguousarray(exp[key]).tobytes(), key


def test_index_determinism(ftk):
  x = cu(np.random.default_rng(3).normal(size=(30000, 48)).astype(np.float32))
  a = ftk.TreeAH(num_leaves=200, dimensions_per_block=3).index(x)
  b = ftk.TreeAH(num_leaves=200, dimensions_per_block=3).index(x)
  for key in INDEX_KEYS:
    assert _np(a._index[key]).tobytes() == _np(b._index[key]).tobytes(), key


# ---- search parity --------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def corpus(ftk):
  x = np.random.default_rng(11).normal(size=(20000, 64)).astype(np.float32)
  return x, tao.build(x, 100, 12, 2)


@pytest.mark.parametrize("probes,reorder,k,Q", [(1, None, 10, 3), (10, None, 100, 4096), (100, None, 256, 1),
                                                (10, 300, 100, 4096), (1, 50, 10, 1), (100, 256, 256, 3),
                                                (10, 1000, 10, 3)])
def test_search_parity(ftk, corpus, probes, reorder, k, Q):
  x, idx = corpus
  q = np.random.default_rng(Q + k).normal(size=(Q, 64)).astype(np.float32)
  layer = ftk.TreeAH(k=k, num_leaves=100, num_leaves_to_search=probes, num_reordering_candidates=reorder).index(cu(x))
  s, i = layer(cu(q))
  _same(s, i, *tao.search(idx, x, q, k, probes, 2, reorder))
  # rank-1 query -> [k] results
  s1, i1 = layer(cu(q[0]))
  assert s1.shape == (k,) and i1.shape == (k,)
  _same(s1, i1, _np(s)[0], _np(i)[0])


def _parity(ftk, x, q, **kw):
  layer = ftk.TreeAH(**kw).index(cu(x))
  s, i = layer(cu(q))
  idx = tao.build(x, kw.get("num_leaves", 100), kw.get("training_iterations", 12), kw.get("dimensions_per_block", 2))
  es, ei = tao.search(idx, x, q, kw.get("k", 10), kw.get("num_leaves_to_search", 10), kw.get("dimensions_per_block", 2),
                      kw.get("num_reordering_candidates"))
  _same(s, i, es, ei)
  return _np(s), _np(i), layer


def test_nan_padding(ftk):
  x = np.random.default_rng(5).normal(size=(300, 16)).astype(np.float32)
  q = np.random.default_rng(6).normal(size=(5, 16)).astype(np.float32)
  s, i, _ = _parity(ftk, x, q, k=30, num_leaves=100, num_leaves_to_search=2)
  assert np.isnan(s).any() and np.all(i[np.isnan(s)] == 0)
  s, i, _ = _parity(ftk, x, q, k=30, num_leaves=100, num_leaves_to_search=2, num_reordering_candidates=40)
  assert np.isnan(s).any() and np.all(i[np.isnan(s)] == 0)


def test_zero_query_and_duplicate_rows(ftk):
  base = np.random.default_rng(8).normal(size=(500, 20)).astype(np.float32)
  x = np.concatenate([base, base, base[:100]])
  q = np.concatenate([np.zeros((1, 20), np.float32), base[:4]])
  for reorder in (None, 64):
    _parity(ftk, x, q, k=20, num_leaves=30, num_leaves_to_search=3, num_reordering_candidates=reorder,
            dimensions_per_block=3)


def test_more_leaves_than_rows(ftk):
  x = np.random.default_rng(9).normal(size=(50, 8)).astype(np.float32)
  q = np.random.default_rng(10).normal(size=(6, 8)).astype(np.float32)
  _parity(ftk, x, q, k=10, num_leaves=100, num_leaves_to_search=20)


def test_query_with_exclusions(ftk):
  x = np.random.default_rng(12).normal(size=(5000, 32)).astype(np.float32)
  q = np.random.default_rng(13).normal(size=(8, 32)).astype(np.float32)
  layer = ftk.TreeAH(k=10, num_leaves=50, num_leaves_to_search=5, num_reordering_candidates=100).index(cu(x))
  excl = np.random.default_rng(14).integers(0, 5000, size=(8, 4))
  _, top = layer(cu(q))
  excl[:, 0] = _np(top)[:, 0]   # exclude every query's best row
  s, i = layer.query_with_exclusions(cu(q), cu(excl))
  idx = tao.build(x, 50, 12, 2)
  es, ei = orc.query_with_exclusions(lambda qq, kk: tao.search(idx, x, qq, kk, 5, 2, 100), q, excl, 10)
  _same(s, i, es, ei)


def test_recall_on_clustered_corpus(ftk):
  """Gaussian mixture: 64 clusters (centers N(0, 9)) of N(0, 1) noise, 20000 x 32, 200 queries drawn the same way,
  num_leaves=100, num_leaves_to_search=10, dimensions_per_block=2, k=10.  The CPU oracle's recall@10 against BruteForce
  is 0.675 without reordering and 1.0 with 100 reordering candidates; the floors below sit under those."""
  rng = np.random.default_rng(7)
  centers = rng.normal(size=(64, 32)).astype(np.float32) * 3
  x = (centers[rng.integers(0, 64, 20000)] + rng.normal(size=(20000, 32)).astype(np.float32)).astype(np.float32)
  q = (centers[rng.integers(0, 64, 200)] + rng.normal(size=(200, 32)).astype(np.float32)).astype(np.float32)
  bf = _np(ftk.BruteForce(k=10).index(cu(x))(cu(q))[1])
  for reorder, floor in ((None, 0.6), (100, 0.95)):
    _, i, _ = _parity(ftk, x, q, k=10, num_reordering_candidates=reorder)
    recall = np.mean([len(set(i[r]) & set(bf[r])) / 10 for r in range(len(q))])
    assert recall >= floor, (reorder, recall)


def test_extra_state_restores_identical_results(ftk):
  x = cu(np.random.default_rng(15).normal(size=(4000, 24)).astype(np.float32))
  q = cu(np.random.default_rng(16).normal(size=(9, 24)).astype(np.float32))
  layer = ftk.TreeAH(k=7, num_leaves=40, num_leaves_to_search=4, num_reordering_candidates=30).index(x, cu(np.arange(4000) * 3))
  restored = ftk.TreeAH(k=7, num_leaves=40, num_leaves_to_search=4, num_reordering_candidates=30)
  restored.load_state_dict(layer.state_dict())
  for a, b in zip(layer(q), restored(q)):
    assert _np(a).tobytes() == _np(b).tobytes()


@pytest.fixture(scope="module")
def few_leaves(ftk):
  x = np.random.default_rng(21).normal(size=(20000, 32)).astype(np.float32)
  return x, tao.build(x, 10, 12, 2)


@pytest.mark.parametrize("probes,reorder,Q", [(1, None, 1), (3, None, 1), (1, 100, 3), (3, 100, 1)])
def test_search_parity_sliced_leaves(ftk, few_leaves, probes, reorder, Q):
  """20000 rows in 10 leaves, Q * probes small: the search cuts every probed leaf into min(ceil(2 * SMs / (Q * probes)),
  rows / L / 256) = 7 slices, so Q = 1 spreads over the SMs; the merged result is still the oracle's."""
  x, idx = few_leaves
  q = np.random.default_rng(22 + Q).normal(size=(Q, 32)).astype(np.float32)
  layer = ftk.TreeAH(k=50, num_leaves=10, num_leaves_to_search=probes, num_reordering_candidates=reorder).index(cu(x))
  s, i = layer(cu(q))
  _same(s, i, *tao.search(idx, x, q, 50, probes, 2, reorder))


def test_search_parity_chunked_queries(ftk, few_leaves):
  """4096 queries x 10 probes x 2048 pre-selected rows do not fit the 512 MB list budget in one piece: the queries run in
  several chunks (7 launches each) and the result is still the oracle's."""
  from recommenders_b200 import ops
  x, idx = few_leaves
  q = np.random.default_rng(23).normal(size=(4096, 32)).astype(np.float32)
  layer = ftk.TreeAH(k=10, num_leaves=10, num_leaves_to_search=10, num_reordering_candidates=2048).index(cu(x))
  tq = cu(q)
  torch.cuda.synchronize()
  before = ops.launch_count()
  s, i = layer(tq)
  torch.cuda.synchronize()
  assert ops.launch_count() - before >= 14
  _same(s, i, *tao.search(idx, x, q, 10, 10, 2, 2048))


def test_index_is_checked_against_queries_and_restores(ftk):
  x = cu(np.random.default_rng(24).normal(size=(3000, 24)).astype(np.float32))
  q = cu(np.random.default_rng(25).normal(size=(5, 24)).astype(np.float32))
  layer = ftk.TreeAH(k=10, num_leaves=20, dimensions_per_block=3, num_reordering_candidates=40).index(x)
  for bad in (cu(np.zeros((5, 32), np.float32)), cu(np.zeros((5, 16), np.float32)), cu(np.zeros(25, np.float32))):
    with pytest.raises(ValueError):
      layer(bad)
  with pytest.raises(ValueError):
    layer(q, k=4096)
  # a layer constructed with another dimensions_per_block searches with the restored index's own block size
  other = ftk.TreeAH(k=10, num_leaves=20, dimensions_per_block=8, num_reordering_candidates=40)
  other.load_state_dict(layer.state_dict())
  for a, b in zip(layer(q), other(q)):
    assert _np(a).tobytes() == _np(b).tobytes()
  # the reordering rows are part of the saved index: a layer set up the other way refuses it
  with pytest.raises(ValueError):
    ftk.TreeAH(k=10, num_leaves=20, dimensions_per_block=3).load_state_dict(layer.state_dict())
