"""Multi-interest (maxsim) retrieval on the GPU against tests/maxsim_oracle.py: K26's head merge on crafted lists
(through `ops` and the C ABI), `BruteForce` with [Q, H, d] queries on the exact and the tensor-core scan, `Streaming`,
`query_with_exclusions`, `FactorizedTopK` and every error path.  Ids and score bits are exact everywhere; the metric
ratios match the oracle's float32 sums to 1e-6."""
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import maxsim_oracle as mo  # noqa: E402

pytestmark = pytest.mark.gpu

F32 = np.float32


@pytest.fixture(scope="module")
def ops():
  from recommenders_b200 import ops as o
  return o


@pytest.fixture(scope="module")
def ftk():
  from recommenders_b200.layers import factorized_top_k as f
  return f


def _dev(a):
  return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _eq(got_s, got_i, want_s, want_i, msg=""):
  gi = got_i.cpu().numpy() if isinstance(got_i, torch.Tensor) else np.asarray(got_i)
  np.testing.assert_array_equal(gi, want_i, err_msg=msg)
  np.testing.assert_array_equal(got_s.cpu().numpy().view(np.uint32), np.asarray(want_s, F32).view(np.uint32), err_msg=msg)


def _normal_case(Q, H, N, d, seed):
  """Normal floats with a duplicate corpus row and a duplicate head (the last head copies head 0)."""
  rs = np.random.RandomState(seed)
  q = rs.normal(size=(Q, H, d)).astype(F32)
  c = rs.normal(size=(N, d)).astype(F32)
  c[N // 2] = c[1]
  if H >= 2:
    q[:, H - 1] = q[:, 0]
  return q, c


# ------------------------------------------------------------------------------------------------
# K26 on crafted lists
# ------------------------------------------------------------------------------------------------
def _lists(Q, H, w, mode, seed):
  """[Q, H, w] per-head lists sorted by (score desc, index asc), distinct indices per list, int64 indices above 2^32.
  all      : every list holds the same w candidates (in its own order)
  disjoint : no candidate is in two lists
  overlap  : each list draws w of 2w candidates
  tie      : as overlap, and candidate 0 sits in every list at a score of +-0 (sign by head), with ties around it"""
  rs = np.random.RandomState(seed)
  s = np.empty((Q, H, w), F32); ix = np.empty((Q, H, w), np.int64)
  for q in range(Q):
    for h in range(H):
      if mode == "all":
        cand = rs.permutation(w)
      elif mode == "disjoint":
        cand = h * w + rs.permutation(w)
      else:
        cand = rs.permutation(2 * w)[:w]
      sc = (rs.randint(-6, 7, size=w) * 0.5).astype(F32)
      if mode == "tie":
        if 0 not in cand:
          cand[0] = 0
        sc[cand == 0] = F32(-0.0) if (h + q) % 2 else F32(0.0)
        sc[rs.rand(w) < 0.2] = F32(0.0)
      gi = (cand.astype(np.int64) * 7919 + 3) << 20
      order = np.lexsort((gi, -sc.astype(np.float64)))
      s[q, h], ix[q, h] = sc[order], gi[order]
  return s, ix


@pytest.mark.parametrize("mode", ["all", "disjoint", "overlap", "tie"])
@pytest.mark.parametrize("H", [1, 2, 3, 32])
@pytest.mark.parametrize("w", [1, 31, 32, 33, 256])
def test_merge_crafted_lists(ops, w, H, mode):
  s, ix = _lists(3, H, w, mode, seed=w * 100 + H)
  ds, di = _dev(s), _dev(ix)
  for k in sorted({1, w}):
    es, ei = mo.merge_head_lists(s, ix, k)
    gs, gi = ops.maxsim_merge(ds, di, k)
    _eq(gs, gi, es, ei, f"{mode} H={H} w={w} k={k}")


@pytest.mark.parametrize("H,w", [(32, 256), (8192, 1), (1, 8192), (2, 4096)])
def test_merge_at_the_entry_limit(ops, H, w):
  s, ix = _lists(2, H, w, "overlap", seed=H + w)
  for k in sorted({1, w}):
    es, ei = mo.merge_head_lists(s, ix, k)
    _eq(*ops.maxsim_merge(_dev(s), _dev(ix), k), es, ei, f"H={H} w={w} k={k}")


def test_merge_above_the_limit_is_rejected(ops):
  for H, w in ((8193, 1), (33, 256)):
    s, ix = torch.zeros((1, H, w), device="cuda"), torch.arange(H * w, device="cuda").reshape(1, H, w)
    with pytest.raises(NotImplementedError, match=f"H={H}"):
      ops.maxsim_merge(s, ix, 1)


def test_merge_through_the_c_abi(ops):
  from recommenders_b200 import _ffi
  for Q, H, w, k_out in ((5, 3, 33, 33), (4, 32, 256, 1), (2, 1, 7, 4)):
    s, ix = _lists(Q, H, w, "tie", seed=Q * H)
    ds, di = _dev(s), _dev(ix)
    out_s = torch.full((Q, k_out), float("nan"), device="cuda"); out_i = torch.full((Q, k_out), -1, dtype=torch.int64, device="cuda")
    rc = _ffi.lib().tfrs_topk_maxsim_merge_f32(_ffi.ptr(ds), _ffi.ptr(di), Q, H, w, k_out, _ffi.ptr(out_s), _ffi.ptr(out_i),
                                               _ffi.stream())
    assert rc == 0, _ffi.last_error()
    es, ei = mo.merge_head_lists(s, ix, k_out)
    _eq(out_s, out_i, es, ei)
  assert _ffi.lib().tfrs_topk_maxsim_merge_f32(_ffi.ptr(ds), _ffi.ptr(di), 1, 8193, 1, 1, _ffi.ptr(out_s), _ffi.ptr(out_i),
                                               _ffi.stream()) == -2
  assert "H=8193" in _ffi.last_error()


def test_rowwise_maxsim(ops):
  for R, H, d in ((1000, 4, 3), (257, 1, 64), (300, 32, 129)):
    q, c = mo.planted_case(R, H, R, d, seed=R + H)
    got = ops.rowwise_maxsim(_dev(q), _dev(c)).cpu().numpy()
    np.testing.assert_array_equal(got.view(np.uint32), mo.rowwise_maxsim(q, c).view(np.uint32))
  one = mo.planted_case(50, 1, 50, 8, seed=3)
  np.testing.assert_array_equal(ops.rowwise_maxsim(_dev(one[0]), _dev(one[1])).cpu().numpy().view(np.uint32),
                                ops.rowwise_dot(_dev(one[0][:, 0]), _dev(one[1])).cpu().numpy().view(np.uint32))


# ------------------------------------------------------------------------------------------------
# BruteForce with [Q, H, d] queries
# ------------------------------------------------------------------------------------------------
EXACT_N, TC_N = 3000, 70000


def _bf(ftk, c, identifiers=None, **kw):
  return ftk.BruteForce(**kw).index(_dev(c), identifiers)


@pytest.mark.parametrize("d", [1, 33, 64, 128, 129])
@pytest.mark.parametrize("route", ["exact", "tc"])
def test_brute_force_d(ops, ftk, route, d):
  N = EXACT_N if route == "exact" else TC_N
  q, c = (mo.planted_case if route == "exact" else _normal_case)(6, 4, N, d, seed=d)
  layer = _bf(ftk, c)
  assert ops.uses_tc_scan(24, N, d, 10) == (route == "tc" and d <= 128)
  es, ei = mo.brute_force(q, c, 10)
  _eq(*layer(_dev(q), k=10), es, ei)


@pytest.mark.parametrize("H", [1, 2, 4, 8, 32])
@pytest.mark.parametrize("k", [1, 10, 100, 256])
@pytest.mark.parametrize("route", ["exact", "tc"])
def test_brute_force_k_h(ops, ftk, route, k, H):
  N = EXACT_N if route == "exact" else TC_N
  q, c = (mo.planted_case if route == "exact" else _normal_case)(5, H, N, 16, seed=k * 100 + H)
  layer = _bf(ftk, c)
  assert ops.uses_tc_scan(5 * H, N, 16, k) == (route == "tc")
  es, ei = mo.brute_force(q, c, k)
  _eq(*layer(_dev(q), k=k), es, ei, f"k={k} H={H}")


@pytest.mark.parametrize("route", ["exact", "tc"])
def test_brute_force_chunks_queries(ops, ftk, route):
  """Q * H head rows well past TC_MAX_Q_PER_CALL: queries go to the scan max(1, 8192 // H) at a time."""
  H = 32
  Q = ops.TC_MAX_Q_PER_CALL // H * 2 + 3
  N = 2000 if route == "exact" else ops.TC_MIN_N
  q, c = _normal_case(Q, H, N, 8, seed=7)
  es, ei = mo.brute_force(q, c, 10)
  _eq(*_bf(ftk, c)(_dev(q), k=10), es, ei)


@pytest.mark.parametrize("route", ["exact", "tc"])
def test_brute_force_identifiers_and_query_model(ftk, route):
  N = EXACT_N if route == "exact" else TC_N
  q, c = _normal_case(7, 3, N, 32, seed=1)
  es, ei = mo.topk_maxsim(q, c, 20)
  ids_t = (torch.arange(N, device="cuda", dtype=torch.int64) * 3 + 11)
  s, i = _bf(ftk, c, ids_t)(_dev(q), k=20)
  _eq(s, i, es, ids_t.cpu().numpy()[ei])
  names = np.array([f"item{j}" for j in range(N)])
  s, i = _bf(ftk, c, names)(_dev(q), k=20)
  _eq(s, i, es, names[ei])
  heads = torch.nn.Linear(32, 3 * 32, bias=False).cuda()
  model = lambda x: heads(x).reshape(-1, 3, 32)   # noqa: E731 -- a query tower that emits three heads
  x = torch.randn(7, 32, device="cuda")
  with torch.no_grad():
    q3 = model(x).contiguous()
    s, i = _bf(ftk, c, query_model=model)(x, k=20)
  es, ei = mo.brute_force(q3.cpu().numpy(), c, 20)
  _eq(s, i, es, ei)


@pytest.mark.parametrize("route", ["exact", "tc"])
def test_one_head_and_equal_heads_give_the_2d_bits(ftk, route):
  N = EXACT_N if route == "exact" else TC_N
  q, c = _normal_case(9, 1, N, 64, seed=2)
  layer = _bf(ftk, c)
  s2, i2 = layer(_dev(q[:, 0]), k=50)
  for q3 in (q, np.repeat(q, 5, axis=1)):
    s3, i3 = layer(_dev(q3), k=50)
    assert torch.equal(i3, i2) and torch.equal(s3.view(torch.int32), s2.view(torch.int32))


# ------------------------------------------------------------------------------------------------
# Streaming, exclusions, FactorizedTopK
# ------------------------------------------------------------------------------------------------
def _streaming(ftk, c, batch, host=False, ids=None, coalesce=None, **kw):
  from recommenders_b200.data import Dataset
  emb = torch.from_numpy(c) if host else _dev(c)
  ds = Dataset.from_tensor_slices(emb if ids is None else (ids, emb)).batch(batch)
  layer = ftk.Streaming(**kw).index_from_dataset(ds)
  if coalesce is not None:
    layer._coalesce_rows = coalesce
  return layer


@pytest.mark.parametrize("host", [False, True])
@pytest.mark.parametrize("N,coalesce", [(EXACT_N, 1000), (TC_N, 20000)])
def test_streaming_equals_brute_force(ftk, N, coalesce, host):
  q, c = _normal_case(6, 4, N, 32, seed=N)
  want = _bf(ftk, c)(_dev(q), k=30)
  es, ei = mo.brute_force(q, c, 30)
  got = _streaming(ftk, c, 512, host=host, coalesce=coalesce, k=30)(_dev(q))
  _eq(*want, es, ei)
  _eq(*got, es, ei)


def test_streaming_short_corpus_and_identifiers(ftk):
  q, c = mo.planted_case(5, 4, 40, 3, seed=9)
  ids = torch.arange(40, device="cuda", dtype=torch.int64) + 1000
  s, i = _streaming(ftk, c, 16, ids=ids, k=100)(_dev(q))   # k > N: min(k, N) entries
  es, ei = mo.topk_maxsim(q, c, 100)
  _eq(s, i, es, ei + 1000)


@pytest.mark.parametrize("route", ["exact", "tc"])
def test_query_with_exclusions(ftk, route):
  N = EXACT_N if route == "exact" else TC_N
  q, c = _normal_case(8, 4, N, 32, seed=4)
  _, top = mo.topk_maxsim(q, c, 12)
  excl = np.concatenate([top[:, ::3], np.full((8, 1), N + 5)], 1).astype(np.int64)   # listed ids and a miss
  es, ei = mo.exclude(q, c, excl, 10)
  _eq(*_bf(ftk, c).query_with_exclusions(_dev(q), _dev(excl), k=10), es, ei)
  _eq(*_streaming(ftk, c, 4096, coalesce=20000, k=10).query_with_exclusions(_dev(q), _dev(excl), k=10), es, ei)
  ids = np.arange(N, dtype=np.int64) * 2 + 1
  es, ei = mo.exclude(q, c, ids[excl % N], 10, identifiers=ids)
  _eq(*_bf(ftk, c, _dev(ids)).query_with_exclusions(_dev(q), _dev(ids[excl % N]), k=10), es, ei)
  _eq(*_streaming(ftk, c, 4096, ids=_dev(ids), k=10).query_with_exclusions(_dev(q), _dev(ids[excl % N]), k=10), es, ei)


@pytest.mark.parametrize("layer_kind", ["brute_force", "streaming"])
@pytest.mark.parametrize("branch", ["score", "id"])
def test_factorized_top_k(ftk, layer_kind, branch):
  from recommenders_b200 import metrics
  N, Q, H, ks = TC_N, 64, 4, (1, 5, 10, 50, 100)
  q, c = _normal_case(Q, H, N, 32, seed=12)
  rs = np.random.RandomState(3)
  true_ids = rs.randint(0, N, size=Q)
  _, top = mo.topk_maxsim(q, c, 100)
  true_ids[::3] = top[::3, 7]            # some positives inside the top 100, at rank <= 7
  true_ids[1::5] = top[1::5, 0]
  w = rs.rand(Q).astype(F32)
  layer = _bf(ftk, c) if layer_kind == "brute_force" else _streaming(ftk, c, 8192, coalesce=20000, k=100)
  m = metrics.FactorizedTopK(layer, ks=ks)
  kw = {"true_candidate_ids": _dev(true_ids)} if branch == "id" else {}
  m.update_state(_dev(q), _dev(c[true_ids]), sample_weight=_dev(w), **kw)
  m.update_state(_dev(q[:10]), _dev(c[true_ids[:10]]), **({"true_candidate_ids": _dev(true_ids[:10])} if kw else {}))
  want_a = mo.factorized_top_k_update(q, c, c[true_ids], ks, true_ids=true_ids if kw else None, sample_weight=w)
  want_b = mo.factorized_top_k_update(q[:10], c, c[true_ids[:10]], ks, true_ids=true_ids[:10] if kw else None)
  want = [(a[0] + b[0]) / (a[1] + b[1]) for a, b in zip(want_a, want_b)]
  np.testing.assert_allclose(m.result(), want, rtol=1e-6, atol=0)   # the oracle sums in float32
  assert 0 < m.result()[-1] < 1


# ------------------------------------------------------------------------------------------------
# errors
# ------------------------------------------------------------------------------------------------
def test_errors(ops, ftk):
  q, c = _normal_case(3, 4, 400, 8, seed=0)
  bf = _bf(ftk, c)
  st = _streaming(ftk, c, 128, k=10)
  for layer in (bf, st):
    with pytest.raises(ValueError, match="rank 1, 2 or 3"):
      layer(_dev(q[None]), k=10)
    with pytest.raises(ValueError):
      layer(_dev(q[:, :, :5]), k=10)
  with pytest.raises(ValueError, match="at least k"):
    bf(_dev(q), k=401)
  big = _dev(np.zeros((2, 33, 8), F32))
  with pytest.raises(NotImplementedError, match="H=33"):
    bf(big, k=256)
  with pytest.raises(NotImplementedError, match="H=33"):
    _streaming(ftk, c, 128, k=256)(big)
  bf_small = _bf(ftk, c[:100])
  s, i = bf_small(big, k=100)   # H * min(k, N) = 3300 is inside the limit
  es, ei = mo.brute_force(np.zeros((2, 33, 8), F32), c[:100], 100)
  _eq(s, i, es, ei)
  assert bf.in_top_k_count(_dev(q), torch.zeros(3, device="cuda"), 10) is None
  shard = ftk.BruteForce(k=10)
  shard._set_index(_dev(c), None)
  shard._shard = (0, object())
  with pytest.raises(NotImplementedError, match="index_shard"):
    shard(_dev(q))
  with pytest.raises(ValueError):
    ops.maxsim_merge(_dev(np.zeros((2, 3), F32)), _dev(np.zeros((2, 3), np.int64)), 1)
  with pytest.raises(ValueError):
    ops.maxsim_merge(_dev(np.zeros((2, 3, 4), F32)), _dev(np.zeros((2, 3, 5), np.int64)), 1)
  with pytest.raises(ValueError):
    ops.maxsim_merge(_dev(np.zeros((2, 3, 4), F32)), _dev(np.zeros((2, 3, 4), np.int64)), 0)
  with pytest.raises(ValueError):
    ops.rowwise_maxsim(_dev(q), _dev(c[:4]))
  with pytest.raises(ValueError):
    ops.rowwise_maxsim(_dev(q), _dev(c[:3, :5]))
  with pytest.raises(ValueError):
    ops.topk_maxsim(_dev(q[:, :0]), _dev(c), 5)
  tree = ftk.TreeAH(k=5, num_leaves=4, num_leaves_to_search=2, training_iterations=1).index(_dev(c))
  with pytest.raises(ValueError, match="rank 2 or 1"):
    tree(_dev(q))
