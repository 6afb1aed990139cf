"""The two thresholds of the tensor-core top-K filter (csrc/topk_tc.cu): top-K and exclusion calls filter at the K'-th
largest bin maximum of the sampled pass, K' the binomial-tail rank of filter_bin_rank, and keep the k-th as the
guaranteed threshold thr_safe; a row that misses at K' is filtered again at thr_safe (a retry) before it may take the
exact fallback.  COUNT calls filter at the k-th.

Every case reads the per-row state out of the call's workspace (tfrs_topk_tc_layout, tfrs_topk_tc_retry_layout) and
checks ids and score bits against the CPU oracle and the exact CUDA-core scan.
"""
import ctypes
import math

import numpy as np
import pytest
import torch
from scipy.stats import binom

from test_gpu_topk_tc_edges import E_ACC, E_REL, TILE, _cdiv, _check_topk, _plan, _tc_rows
from oracle import oracle as orc

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ops():
  from recommenders_b200 import ops as o
  return o


def _retry_layout(ops, Q, N, d, k):
  out = (ctypes.c_int64 * 4)()
  ops.check(ops.lib().tfrs_topk_tc_retry_layout(Q, N, d, k, out), "topk_tc_retry_layout")
  return [int(x) for x in out]


def _retry_rows(ops, Q, N, d, k):
  """thr_safe and the retry marks of the most recent call of this shape, as numpy arrays over the Q rows."""
  o_safe, o_retry, _, _ = _retry_layout(ops, Q, N, d, k)
  ws = ops.workspace(0, torch.device("cuda", torch.cuda.current_device()), "tc")
  base = (-ws.data_ptr()) % 16
  torch.cuda.synchronize()
  safe = ws[base + o_safe: base + o_safe + 4 * Q].view(torch.float32).cpu().numpy()
  retry = ws[base + o_retry: base + o_retry + 4 * Q].view(torch.int32).cpu().numpy()
  return safe, retry


def _binomial_rank(k, stride):
  """The smallest K' with P(Binomial(k - 1, 1/stride) >= K') <= 1e-9 (k when every tile is sampled)."""
  if stride == 1:
    return k
  return next(r for r in range(1, k + 1) if binom.sf(r - 1, k - 1, 1.0 / stride) <= 1e-9)


def test_filter_bin_rank_is_the_binomial_tail(ops):
  Q, d = 256, 64
  seen = set()
  for k in range(1, 257):
    for tiles in (2 * k, 4 * k, 32 * k):   # the plan halves the stride 4 while it leaves too few sampled bins
      N = tiles * TILE
      if not ops.tc_supported(Q, N, d, k):
        continue
      _, _, k_filter, stride = _retry_layout(ops, Q, N, d, k)
      assert stride == _plan(Q, N, d, k)["stride"]
      assert k_filter == _binomial_rank(k, stride), (k, stride, k_filter)
      seen.add(stride)
  assert seen == {1, 2, 4}, seen
  assert [_retry_layout(ops, Q, 1 << 20, d, k)[2] for k in (50, 100, 256)] == [33, 54, 109]


def _sampled_bin_max(dots, N, plan):
  """[Q, n_bins] bin maxima of the sampled pass restated from exact scores: each corpus part's sampled tiles in groups
  of `group`, one bin per group and 64-column half."""
  stride, n_sample = plan["stride"], plan["n_sample"]
  parts = min(plan["parts"], n_sample)
  iters_max = _cdiv(n_sample, parts)
  g = 1
  while parts * _cdiv(iters_max, g) * 2 > max(4 * plan["k"], 512) and g < iters_max:
    g += 1
  bins = []
  for p in range(parts):
    u0, u1 = p * n_sample // parts, (p + 1) * n_sample // parts
    for b0 in range(u0, u1, g):
      tiles = np.arange(b0, min(b0 + g, u1)) * stride
      for h in range(2):
        cols = (tiles[:, None] * TILE + 64 * h + np.arange(64)).reshape(-1)
        bins.append(dots[:, cols].max(1))
  return np.stack(bins, 1)


def test_thresholds_at_their_bin_ranks(ops):
  """Small-integer data: every screening score is exact (integer dot product times 2^(corpus + row exponent)), so the
  bin maxima are restated bit for bit.  thr sits at the K'-th of them and thr_safe at the k-th, both lowered by the
  same margin; COUNT filters at the k-th, bit for bit the top-K call's thr_safe."""
  Q, N, d, k = 256, 131072, 64, 100
  g = torch.Generator(device="cuda"); g.manual_seed(31)
  q = torch.randint(-32, 33, (Q, d), generator=g, device="cuda").float()
  c = torch.randint(-32, 33, (N, d), generator=g, device="cuda").float()
  image = ops.index_build(c)
  _check_topk(ops, q, c, k)
  rows = _tc_rows(ops, Q, N, d, k)
  safe, retry = _retry_rows(ops, Q, N, d, k)
  k_filter = _retry_layout(ops, Q, N, d, k)[2]
  assert k_filter == 54
  plan = dict(_plan(Q, N, d, k), k=k)
  dots = q.double().cpu().numpy() @ c.double().cpu().numpy().T
  bm = -np.sort(-_sampled_bin_max(dots, N, plan), axis=1)
  assert bm.shape[1] == rows["n_bins"]
  unit = np.ldexp(1.0, 15 - math.frexp(32.0)[1] + rows["qexp"].astype(np.int64))   # screening units per score unit
  L_k, L_f = bm[:, k - 1] * unit, bm[:, k_filter - 1] * unit
  margin = L_k - safe.astype(np.float64)
  np.testing.assert_allclose(margin, rows["cut"] * (1 + E_ACC / (2 * E_REL)), rtol=1e-4)
  thr = rows["thr"].astype(np.float64)
  tol = np.spacing(np.abs(rows["thr"])).astype(np.float64) + np.spacing(np.abs(safe)).astype(np.float64)
  kept = retry == 0
  assert (np.abs(thr - (L_f - margin)) <= tol)[kept].all(), "thr is the K'-th bin bound"
  np.testing.assert_array_equal(rows["thr"][~kept], safe[~kept])
  ops.topk_tc_count(q, c, image, k, torch.zeros(Q, device="cuda"))
  np.testing.assert_array_equal(_tc_rows(ops, Q, N, d, k)["thr"].view(np.uint32), safe.view(np.uint32))
  np.testing.assert_array_equal(_retry_rows(ops, Q, N, d, k)[0].view(np.uint32), safe.view(np.uint32))


# ------------------------------------------------------------------------------------------------
# planted retries.  Candidates: dims 0 and 1 uniform in [-0.5, 0.5], the rest 0.1 N(0, 1).  K rows hold 1 + 0.01 r
# (r < K) in both dims 0 and 1, each in the first tile of its own bin of the sampled pass, so each is a bin maximum.
# A query e0 then has its k best one per bin: the K'-th bin maximum is its K'-th best, its filter keeps K' < k
# survivors, it retries at the k-th bin maximum and finishes on the tensor cores.  A block of BLOCK rows in unsampled
# tiles holds 1 - 0.0025 in dim 1 (0 in dim 0): below the k-th best of a query e1 but above its thr_safe, so e1 retries
# and then overflows its survivor keys: the exact fallback.  The other queries are random in dims 2.. .
# ------------------------------------------------------------------------------------------------
PQ, PN, PD, PK, PE, BLOCK = 300, 65536, 64, 100, 5, 1200
RETRY_ROWS = np.array([3, 100, 255, 256, 299])    # both 256-query blocks, their first / last rows
FALLBACK_ROWS = np.array([7, 200, 270])


def _planted(seed):
  plan = dict(_plan(PQ, PN, PD, PK), k=PK)
  stride, n_sample = plan["stride"], plan["n_sample"]
  parts = min(plan["parts"], n_sample)
  firsts = []   # the first sampled tile of each bin (one group per part at this shape)
  for p in range(parts):
    u0, u1 = p * n_sample // parts, (p + 1) * n_sample // parts
    iters_max = _cdiv(n_sample, parts)
    g = 1
    while parts * _cdiv(iters_max, g) * 2 > max(4 * PK, 512) and g < iters_max:
      g += 1
    firsts += [u * stride for u in range(u0, u1, g)]
  firsts = np.array(firsts)
  assert 2 * len(firsts) >= PK
  rng = np.random.default_rng(seed)
  members = np.concatenate([firsts * TILE + 5, firsts * TILE + 64 + 9])[rng.permutation(2 * len(firsts))[:PK]]
  sampled = set((np.arange(n_sample) * stride).tolist())
  free = np.array([t for t in range(PN // TILE) if t not in sampled])
  block = free[np.arange(BLOCK) % len(free)] * TILE + 17 + (np.arange(BLOCK) // len(free)) * 3
  cn = np.empty((PN, PD), np.float32)
  cn[:, :2] = rng.uniform(-0.5, 0.5, (PN, 2))
  cn[:, 2:] = 0.1 * rng.standard_normal((PN, PD - 2))
  cn[members, 0] = cn[members, 1] = (1.0 + 0.01 * rng.permutation(PK)).astype(np.float32)
  cn[block, 0] = 0.0
  cn[block, 1] = np.float32(1.0 - 0.0025)
  qn = np.zeros((PQ, PD), np.float32)
  qn[:, 2:] = rng.standard_normal((PQ, PD - 2))
  qn[RETRY_ROWS] = 0.0; qn[RETRY_ROWS, 0] = 1.0
  qn[FALLBACK_ROWS] = 0.0; qn[FALLBACK_ROWS, 1] = 1.0
  return torch.from_numpy(qn).cuda(), torch.from_numpy(cn).cuda()


def _records(ops, Q, N, d, k):
  """count [Q, segs] and each row's live records (index, 8 scores), as the workspace holds them."""
  out = (ctypes.c_int64 * 10)()
  ops.check(ops.lib().tfrs_topk_tc_layout(Q, N, d, k, out), "topk_tc_layout")
  o_count, _, _, o_cand, segs, cap, Qp = [int(x) for x in out[:7]]
  ws = ops.workspace(0, torch.device("cuda", torch.cuda.current_device()), "tc")
  base = (-ws.data_ptr()) % 16
  torch.cuda.synchronize()
  count = ws[base + o_count: base + o_count + 4 * Qp * segs].view(torch.int32).view(Qp, segs)[:Q].cpu().numpy()
  cand_s = ws[base + o_cand: base + o_cand + 32 * Qp * segs * cap].view(torch.int32).view(Qp, segs, cap, 8)[:Q].cpu().numpy()
  o_i = o_cand + 32 * Qp * segs * cap
  cand_i = ws[base + o_i: base + o_i + 4 * Qp * segs * cap].view(torch.int32).view(Qp, segs, cap)[:Q].cpu().numpy()
  live = np.arange(cap)[None, None, :] < np.minimum(count, cap)[:, :, None]
  return count, [(cand_i[r][live[r]], cand_s[r][live[r]]) for r in range(Q)]


def test_planted_retries_topk(ops):
  q, c = _planted(41)
  s, i, rows = _check_topk(ops, q, c, PK, FALLBACK_ROWS)
  safe, retry = _retry_rows(ops, PQ, PN, PD, PK)
  np.testing.assert_array_equal(np.flatnonzero(retry), np.sort(np.concatenate([RETRY_ROWS, FALLBACK_ROWS])),
                                err_msg="the rows that were filtered again at thr_safe")
  # a retried row's workspace holds its thr_safe records: exactly its k planted members survive it
  np.testing.assert_array_equal(rows["thr"][RETRY_ROWS].view(np.uint32), safe[RETRY_ROWS].view(np.uint32))
  np.testing.assert_array_equal(rows["n"][RETRY_ROWS], PK)
  others = np.setdiff1d(np.arange(PQ), np.concatenate([RETRY_ROWS, FALLBACK_ROWS]))
  assert (rows["thr"][others] > safe[others]).all(), "ordinary rows filter above the guaranteed threshold"
  assert (rows["n"][others] >= PK).all()
  # the records of the rows that were not retried do not depend on whether their query block was rescanned: the same
  # rows in a batch without planted queries
  count, rec = _records(ops, PQ, PN, PD, PK)
  q2 = q.clone()
  planted = torch.from_numpy(np.concatenate([RETRY_ROWS, FALLBACK_ROWS])).cuda()
  q2[planted] = q[torch.from_numpy(others[:len(planted)]).cuda()]
  ops.topk_tc(q2, c, ops.index_build(c), PK)
  assert not _retry_rows(ops, PQ, PN, PD, PK)[1].any()
  count2, rec2 = _records(ops, PQ, PN, PD, PK)
  np.testing.assert_array_equal(count[others], count2[others])
  for r in others:
    assert np.array_equal(rec[r][0], rec2[r][0]) and np.array_equal(rec[r][1], rec2[r][1]), r


def test_planted_retries_exclude(ops):
  q, c = _planted(42)
  k = PK - PE                                   # k + E = PK candidates are fetched: the same filter rank
  os_, oi = orc.topk_scan(q.cpu().numpy(), c.cpu().numpy(), PK)
  g = torch.Generator(device="cuda"); g.manual_seed(43)
  ex = torch.randint(0, PN, (PQ, PE), generator=g, device="cuda")
  oi_t = torch.from_numpy(oi).cuda()
  ex[:, 0] = oi_t[:, 0]; ex[:, 1] = oi_t[:, 50]; ex[::2, 2] = oi_t[::2, PK - 1]
  s, i = ops.topk_tc_exclude(q, c, ops.index_build(c), k, ex)
  rows = _tc_rows(ops, PQ, PN, PD, PK)
  np.testing.assert_array_equal(np.flatnonzero(rows["fallback"]), FALLBACK_ROWS)
  np.testing.assert_array_equal(np.flatnonzero(_retry_rows(ops, PQ, PN, PD, PK)[1]),
                                np.sort(np.concatenate([RETRY_ROWS, FALLBACK_ROWS])))
  es_, ei_ = orc.exclude(os_, oi, ex.cpu().numpy(), k)
  np.testing.assert_array_equal(i.cpu().numpy(), ei_)
  np.testing.assert_array_equal(s.cpu().numpy().view(np.uint32), es_.view(np.uint32))


@pytest.mark.parametrize("fill", [0x00, 0xFF, 0x01])
def test_sentinel_filled_workspace(ops, fill):
  """Nothing the call reads is left over from an earlier one: the same state and outputs from any workspace contents
  (0xFF bytes are NaN thresholds and counts above every capacity, 0x01 bytes retry marks on every row)."""
  q, c = _planted(44)
  image = ops.index_build(c)
  ops.topk_tc(q, c, image, PK)
  ops.workspace(0, q.device, "tc").fill_(fill)
  s, i, rows = _check_topk(ops, q, c, PK, FALLBACK_ROWS)
  np.testing.assert_array_equal(np.flatnonzero(_retry_rows(ops, PQ, PN, PD, PK)[1]),
                                np.sort(np.concatenate([RETRY_ROWS, FALLBACK_ROWS])))
