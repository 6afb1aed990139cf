"""GPU parity tests of the tensor-core top-K path (wgmma screening + exact re-scoring), through the C ABI.
Bar: bit-exact ids and scores against the CPU oracle and against the exact CUDA-core path."""
import numpy as np
import pytest
import torch

from oracle import oracle as orc

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ops():
  from recommenders_b200 import ops as o
  return o


def _rand(shape, seed, scale=1.0):
  g = torch.Generator(device="cuda"); g.manual_seed(seed)
  return torch.randn(shape, generator=g, device="cuda") * scale


def _check(ops, q, c, k, offset=0, oracle_rows=32, max_fallback=0):
  idx = ops.index_build(c)
  assert ops.tc_supported(q.shape[0], c.shape[0], c.shape[1], k)
  s, i = ops.topk_tc(q, c, idx, k, index_offset=offset)
  if max_fallback is not None:
    # the tensor-core path itself -- not the exact fallback that backs it up -- must have produced the result
    st = ops.tc_last_call_stats(q.shape[0], c.shape[0], c.shape[1], k)
    assert st["fallback_queries"] <= max_fallback, st
    assert st["survivors_mean"] >= k, st
  es, ei = ops.topk_scan(q, c, k, index_offset=offset)
  assert torch.equal(i, ei) and torch.equal(s, es), "tensor-core path differs from the exact CUDA-core path"
  r = min(oracle_rows, q.shape[0])
  os_, oi = orc.topk_scan(q[:r].cpu().numpy(), c.cpu().numpy(), k, index_offset=offset)
  np.testing.assert_array_equal(i[:r].cpu().numpy(), oi)
  np.testing.assert_array_equal(s[:r].cpu().numpy().view(np.uint32), os_.view(np.uint32))
  return s, i


@pytest.mark.parametrize("Q,N,d,k", [(300, 40000, 64, 100), (256, 32768, 64, 100), (1000, 200000, 128, 10),
                                     (17, 65537, 33, 50), (513, 100001, 100, 128), (4096, 131072, 64, 100),
                                     (1, 300000, 64, 1), (700, 400000, 64, 256)])
def test_tc_matches_exact(ops, Q, N, d, k):
  _check(ops, _rand((Q, d), 2), _rand((N, d), 1), k)


def test_tc_index_offset_and_negative_scores(ops):
  # all scores negative and N not a multiple of 128: zero-padded rows must never be returned
  c = torch.rand((50001, 64), device="cuda") + 0.1
  q = -(torch.rand((64, 64), device="cuda") + 0.1)
  s, i = _check(ops, q, c, 20, offset=123456789, max_fallback=None)  # narrow score spread: wide band, fallback allowed
  assert int(i.min()) >= 123456789 and int(i.max()) < 123456789 + 50001 and float(s.max()) < 0


def test_tc_ties_overflow_fallback(ops):
  # every candidate identical -> every screening score ties -> survivor lists overflow -> exact fallback
  c = torch.ones((40000, 64), device="cuda"); q = _rand((40, 64), 3)
  s, i = _check(ops, q, c, 10, max_fallback=None)  # every query must take the exact fallback here
  assert ops.tc_last_call_stats(40, 40000, 64, 10)["fallback_queries"] == 40
  assert torch.equal(i, torch.arange(10, device="cuda").expand(40, 10))
  # duplicated corpus blocks: exact duplicates across tiles, lowest index must win
  base = _rand((20000, 64), 4)
  _check(ops, _rand((100, 64), 5), torch.cat([base, base, base], 0), 30, max_fallback=None)


def test_tc_scaled_inputs(ops):
  # large dynamic range: margins scale with |q| * max|c|
  _check(ops, _rand((128, 64), 6, 1e3), _rand((60000, 64), 7, 1e-3), 25)
  c = _rand((60000, 64), 8); c[12345] *= 1000.0   # one huge-norm row inflates the bound -> more survivors, same answer
  _check(ops, _rand((64, 64), 9), c, 10, max_fallback=None)


def test_tc_full_size_properties(ops):
  """BASELINE config 2 at full size (1M x 64, 4096 queries, top-100): size-independent properties +
  exact-path equality on a slice + oracle on a few rows."""
  N, d, Q, k = 1_000_000, 64, 4096, 100
  c = _rand((N, d), 1); q = _rand((Q, d), 2)
  idx = ops.index_build(c)
  s, i = ops.topk_tc(q, c, idx, k)
  st = ops.tc_last_call_stats(Q, N, d, k)
  assert st["fallback_queries"] == 0 and st["survivors_mean"] >= k, st
  assert bool((s[:, :-1] >= s[:, 1:]).all()), "scores must be sorted descending"
  assert int(i.min()) >= 0 and int(i.max()) < N
  assert all(len(set(r)) == k for r in i[:64].cpu().tolist()), "indices must be distinct"
  # returned scores are the exact chain of the returned rows
  rows = torch.arange(0, Q, 37, device="cuda")
  for j in (0, 57, 99):
    assert torch.equal(ops.rowwise_dot(q[rows], c[i[rows, j]]), s[rows, j])
  es, ei = ops.topk_scan(q[:256], c, k)
  assert torch.equal(i[:256], ei) and torch.equal(s[:256], es)
  os_, oi = orc.topk_scan(q[4000:4008].cpu().numpy(), c.cpu().numpy(), k)
  np.testing.assert_array_equal(i[4000:4008].cpu().numpy(), oi)
  np.testing.assert_array_equal(s[4000:4008].cpu().numpy(), os_)


def test_bruteforce_layer_uses_tc_and_shards(ops):
  import recommenders_b200 as tfrs
  c = _rand((70000, 64), 11); q = _rand((200, 64), 12)
  layer = tfrs.layers.factorized_top_k.BruteForce(k=50).index(c)
  assert layer._tc_index is not None
  s, i = layer(q)
  es, ei = ops.topk_scan(q, c, 50)
  assert torch.equal(i.to(torch.int64), ei) and torch.equal(s, es) and i.dtype == torch.int32
  # emulate the 2-shard protocol in one process: local scans with offsets, then the merge kernel
  parts = []
  for lo, hi in (tfrs.layers.factorized_top_k.shard_bounds(70000, r, 2) for r in range(2)):
    l = tfrs.layers.factorized_top_k.BruteForce(k=50).index(c[lo:hi])
    parts.append(l._local_topk(q, 50, lo))
  ms, mi = ops.topk_merge(torch.stack([p[0] for p in parts]), torch.stack([p[1] for p in parts]), 50)
  assert torch.equal(mi, ei) and torch.equal(ms, es)


def test_packed_allgather_block_merge(ops):
  """The merge kernel reads the all-gather receive buffer in place: blocks of [scores f32 | pad | indices i64]."""
  import recommenders_b200 as tfrs
  c = _rand((90000, 64), 21); q = _rand((333, 64), 22); k = 100
  es, ei = ops.topk_scan(q, c, k)
  Q = q.shape[0]
  idx_off = (Q * k * 4 + 7) // 8 * 8
  block = idx_off + Q * k * 8
  world = 3
  recv = torch.empty(world * block, dtype=torch.uint8, device="cuda")
  for r in range(world):
    lo, hi = tfrs.layers.factorized_top_k.shard_bounds(90000, r, world)
    blk = recv[r * block:(r + 1) * block]
    out_s = blk[:Q * k * 4].view(torch.float32).view(Q, k); out_i = blk[idx_off:].view(torch.int64).view(Q, k)
    layer = tfrs.layers.factorized_top_k.BruteForce(k=k).index(c[lo:hi])
    layer._local_topk(q, k, lo, out=(out_s, out_i))
  ms, mi = ops.topk_merge_packed(recv, world, Q, k, k, idx_off, block)
  assert torch.equal(mi, ei) and torch.equal(ms, es)


def test_tc_query_chunking(ops):
  """More queries than TC_MAX_Q_PER_CALL: the wrapper runs query chunks into slices of one output."""
  c = _rand((40000, 64), 31); q = _rand((9001, 64), 32)
  idx = ops.index_build(c)
  s, i = ops.topk_tc(q, c, idx, 10)
  es, ei = ops.topk_scan(q[-300:], c, 10)
  assert torch.equal(i[-300:], ei) and torch.equal(s[-300:], es)
  es, ei = ops.topk_scan(q[8000:8300], c, 10)
  assert torch.equal(i[8000:8300], ei) and torch.equal(s[8000:8300], es)


@pytest.mark.parametrize("world,Q,k_in,k", [(2, 37, 100, 100), (8, 300, 100, 100), (5, 64, 16, 50), (3, 10, 7, 21), (8, 5, 256, 256), (7, 20, 10, 64), (1, 9, 12, 12)])
def test_sorted_merge_equals_sorting_merge(ops, world, Q, k_in, k):
  """Rank-by-binary-search merge of sorted per-shard lists == the generic sort-based merge == numpy lexsort, with
  heavy score ties (quantised scores), tied scores across lists and (-inf, INT64_MAX) padding of short shards."""
  rng = np.random.default_rng(world * 1000 + Q)
  idx_off = (Q * k_in * 4 + 7) // 8 * 8
  block = idx_off + Q * k_in * 8
  recv = torch.zeros(world * block, dtype=torch.uint8, device="cuda")
  all_s = np.empty((world, Q, k_in), np.float32); all_i = np.empty((world, Q, k_in), np.int64)
  for r in range(world):
    s = np.round(rng.normal(size=(Q, k_in)) * 2).astype(np.float32) / 2       # many exact ties
    i = np.stack([rng.choice(1000, size=k_in, replace=False) for _ in range(Q)]).astype(np.int64) + 1000 * r
    n_pad = int(rng.integers(0, k_in // 2 + 1)) if r == world - 1 else 0         # a short last shard
    if n_pad:
      s[:, k_in - n_pad:] = -np.inf; i[:, k_in - n_pad:] = np.iinfo(np.int64).max
    order = np.lexsort((i, -s), axis=1)                                          # (score desc, index asc) per list
    s = np.take_along_axis(s, order, 1); i = np.take_along_axis(i, order, 1)
    all_s[r], all_i[r] = s, i
    blk = recv[r * block:(r + 1) * block]
    blk[:Q * k_in * 4].view(torch.float32).view(Q, k_in).copy_(torch.from_numpy(s))
    blk[idx_off:].view(torch.int64).view(Q, k_in).copy_(torch.from_numpy(i))
  fs, fi = ops.topk_merge_packed(recv, world, Q, k_in, k, idx_off, block, sorted_lists=True)
  gs, gi = ops.topk_merge_packed(recv, world, Q, k_in, k, idx_off, block, sorted_lists=False)
  cs = all_s.transpose(1, 0, 2).reshape(Q, -1); ci = all_i.transpose(1, 0, 2).reshape(Q, -1)
  order = np.lexsort((ci, -cs), axis=1)[:, :k]
  es = np.take_along_axis(cs, order, 1); ei = np.take_along_axis(ci, order, 1)
  np.testing.assert_array_equal(fs.cpu().numpy(), es); np.testing.assert_array_equal(fi.cpu().numpy(), ei)
  assert torch.equal(fs, gs) and torch.equal(fi, gi)
