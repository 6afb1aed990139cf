"""Edge cases of the tensor-core top-K scan (csrc/topk_tc.cu): the exact fallbacks of all three finalize modes (TOPK,
EXCLUDE, COUNT) in batches that mix fallback and tensor-core rows, the shape boundaries of the scan, the selection and
threshold branches, COUNT positives at the filter threshold, and per-row magnitude and signed-zero edges.

Every case checks ids and score BIT PATTERNS against the CPU oracle (the canonical fmaf chain from +0.0f, so -0.0f is
a score of its own that ranks equal to +0.0f), the same bits against the exact CUDA-core scan, and exactly which rows
took the exact fallback, read per row out of the call's workspace.

NaN in queries or candidates is out of scope: the oracle's (score desc, index asc) order is not total for NaN scores.
NaN positives of the COUNT mode are in scope (no score is above NaN).
"""
import ctypes
import math

import numpy as np
import pytest
import torch

from oracle import oracle as orc

pytestmark = pytest.mark.gpu

TILE = 128                  # corpus rows per screening tile
ORACLE_FMA_BUDGET = 1.5e9   # above Q * N * d the oracle checks a stated sample of rows (which always holds the planted ones)


@pytest.fixture(scope="module")
def ops():
  from recommenders_b200 import ops as o
  return o


def _rand(shape, seed, scale=1.0):
  g = torch.Generator(device="cuda"); g.manual_seed(seed)
  return torch.randn(shape, generator=g, device="cuda") * scale


def _cdiv(a, b):
  return -(-a // b)


def _bits(t):
  return t.contiguous().view(torch.int32)


def _plan(Q, N, d, k):
  """make_plan (csrc/topk_tc.cu) restated for the quantities that pick a branch: sample stride, bins of the sampled
  pass, survivor segments and their capacity, and the finalize capacities (survivor keys, re-scored band)."""
  sms = torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count
  full_tiles = N // TILE
  stride = 4
  while stride > 1 and 2 * _cdiv(full_tiles, stride) < 4 * k:
    stride >>= 1
  n_sample = _cdiv(full_tiles, stride)
  parts = min(max(sms // _cdiv(Q, 256), 1), 132)
  parts_sample = min(parts, n_sample)
  parts_full = min(parts, _cdiv(N, TILE))
  iters_max = _cdiv(n_sample, parts_sample)
  g = 1
  while parts_sample * _cdiv(iters_max, g) * 2 > max(4 * k, 512) and g < iters_max:
    g += 1
  lam = k * stride / (parts_full * 2.0)
  cap_part = 32
  while cap_part < 2.0 * lam + 12.0 * math.sqrt(lam) + 8.0 and cap_part < 512:
    cap_part <<= 1
  cap_keys = 1024
  while cap_keys < 1.6 * 1.3 * k * stride and cap_keys < 4096:
    cap_keys <<= 1
  return {"stride": stride, "n_sample": n_sample, "n_bins": parts_sample * _cdiv(iters_max, g) * 2, "parts": parts,
          "segs": 2 * parts_full, "cap_part": cap_part, "cap_keys": cap_keys, "cap_band": cap_keys // 2}


def _tc_rows(ops, Q, N, d, k):
  """Per-row state of the most recent tensor-core call of this shape, read out of its workspace at the offsets
  tfrs_topk_tc_layout reports (as ops.tc_last_call_stats does), as numpy arrays over the Q rows:
    fallback  the row took the exact fallback
    seg_ovf   one of its survivor segments overflowed in the filter pass
    records   octet records in its survivor lists (what the select kernel's 13-bit record locator indexes)
    n         screening scores >= its filter threshold in those records: the survivors the select kernel ranks
    thr, cut  its filter threshold and re-scored band width (screening units)
    qexp      its power-of-two rescale exponent (screening score = score * 2^(corpus exponent + qexp))
  and n_bins, the bin count of the sampled pass (> 512 selects tc_threshold_kernel<32>).  The restated plan is checked
  against the library's layout."""
  out = (ctypes.c_int64 * 10)()
  ops.check(ops.lib().tfrs_topk_tc_layout(Q, N, d, k, out), "topk_tc_layout")
  o_count, o_ovf, o_thr, o_cand, segs, cap, Qp, o_cut, n_bins, o_qexp = [int(x) for x in out]
  plan = _plan(Q, N, d, k)
  assert (plan["segs"], plan["cap_part"], plan["n_bins"]) == (segs, cap, n_bins), (plan, segs, cap, n_bins)
  dev = torch.device("cuda", torch.cuda.current_device())
  ws = ops.workspace(0, dev, "tc")
  base = (-ws.data_ptr()) % 16
  torch.cuda.synchronize()

  def arr(off, n, dtype):   # every array read here has 4-byte elements
    return ws[base + off: base + off + 4 * n].view(dtype)

  count = arr(o_count, Qp * segs, torch.int32).view(Qp, segs)[:Q].to(torch.int64)
  ovf = arr(o_ovf, Q, torch.int32)
  thr = arr(o_thr, Q, torch.float32)
  cand_s = arr(o_cand, Qp * segs * cap * 8, torch.float32).view(Qp, segs, cap, 8)[:Q]
  cand_i = arr(o_cand + Qp * segs * cap * 32, Qp * segs * cap, torch.int32).view(Qp, segs, cap)[:Q]
  live = torch.arange(cap, device=dev)[None, None, :] < count.clamp(max=cap)[:, :, None]
  col = cand_i.to(torch.int64)[..., None] + torch.arange(8, device=dev)
  surv = (cand_s >= thr[:, None, None, None]) & live[..., None] & (col < N)
  return {"fallback": (ovf != 0).cpu().numpy(), "seg_ovf": (count > cap).any(1).cpu().numpy(),
          "records": count.clamp(max=cap).sum(1).cpu().numpy(), "n": surv.flatten(1).sum(1).cpu().numpy(),
          "thr": thr.cpu().numpy(), "cut": arr(o_cut, Q, torch.float32).cpu().numpy(),
          "qexp": arr(o_qexp, Q, torch.int32).cpu().numpy(), "n_bins": n_bins}


def _assert_fallback(rows, expected):
  np.testing.assert_array_equal(np.flatnonzero(rows["fallback"]), np.sort(np.asarray(expected, np.int64)),
                                err_msg="the rows that took the exact fallback")


def _oracle_rows(Q, N, d, must=()):
  """Every row when the oracle can afford it, else 64 evenly spaced rows plus every row in `must`."""
  if Q * N * d <= ORACLE_FMA_BUDGET:
    return np.arange(Q)
  return np.union1d(np.linspace(0, Q - 1, 64).astype(np.int64), np.asarray(must, np.int64))


def _check_topk(ops, q, c, k, fallback_rows=(), index_offset=0):
  """topk_tc on (q, c): the exact set of fallback rows, ids and score bits == the oracle and == topk_scan."""
  Q, d = q.shape; N = c.shape[0]
  assert ops.tc_supported(Q, N, d, k), (Q, N, d, k)
  s, i = ops.topk_tc(q, c, ops.index_build(c), k, index_offset=index_offset)
  rows = _tc_rows(ops, Q, N, d, k)
  _assert_fallback(rows, fallback_rows)
  r = _oracle_rows(Q, N, d, fallback_rows)
  os_, oi = orc.topk_scan(q[torch.from_numpy(r).cuda()].cpu().numpy(), c.cpu().numpy(), k, index_offset=index_offset)
  np.testing.assert_array_equal(i[torch.from_numpy(r).cuda()].cpu().numpy(), oi)
  np.testing.assert_array_equal(s[torch.from_numpy(r).cuda()].cpu().numpy().view(np.uint32), os_.view(np.uint32))
  es, ei = ops.topk_scan(q, c, k, index_offset=index_offset)
  assert torch.equal(i, ei) and torch.equal(_bits(s), _bits(es)), "tensor-core path differs from the exact CUDA-core path"
  return s, i, rows


def _count_expected(full, pos, k):
  """min(k, #{candidates scoring strictly above the positive}) on the oracle's [Q, N] scores."""
  return np.minimum((full > pos[:, None]).sum(1), k)


# ------------------------------------------------------------------------------------------------
# 1. mixed batches: fallback rows planted among tensor-core rows, all three finalize modes
# ------------------------------------------------------------------------------------------------
# Candidates: random rows with dimension 0 zeroed, plus a block of V identical rows v = A e0.  A query with a large q0
# scores the whole block at q0 A, far above every random row: thousands of exact ties at the top overflow its survivor
# keys / re-scored band and it takes the exact fallback.  A query with q0 = 0 scores v at exactly 0, far below its
# top-k, and stays on the tensor-core path.  32768 rows = 256 tiles over 66 corpus parts (two 256-query blocks) keep
# every survivor segment within its 32 records, so the survivor keys (TOPK, EXCLUDE) or the COUNT band overflow, not a
# segment.
MIX_Q, MIX_N, MIX_D, MIX_K, MIX_E = 300, 32768, 64, 50, 5
MIX_V0, MIX_V, MIX_A = 8000, 2048, 8.0
MIX_FALLBACK = np.array([0, 1, 7, 100, 254, 255, 256, 257, 298, 299])   # first / last row, both sides of a 256-query block


@pytest.fixture(scope="module")
def mixed(ops):
  c = _rand((MIX_N, MIX_D), 101)
  c[:, 0] = 0.0
  c[MIX_V0:MIX_V0 + MIX_V] = 0.0
  c[MIX_V0:MIX_V0 + MIX_V, 0] = MIX_A
  q = _rand((MIX_Q, MIX_D), 102)
  q[:, 0] = 0.0
  fb = torch.from_numpy(MIX_FALLBACK).cuda()
  q[fb, 0] = 6.0 + 0.5 * (fb % 5).float()      # ties at q0 A in [48, 64]: every random row scores below ~35
  return q, c, ops.index_build(c)


def test_mixed_fallback_topk(ops, mixed):
  import recommenders_b200 as tfrs
  q, c, _ = mixed
  s, i, _ = _check_topk(ops, q, c, MIX_K, MIX_FALLBACK)
  fb = torch.from_numpy(MIX_FALLBACK).cuda()
  assert torch.equal(i[fb], torch.arange(MIX_V0, MIX_V0 + MIX_K, device="cuda").expand(len(fb), MIX_K))
  assert torch.equal(s[fb], (q[fb, 0] * MIX_A)[:, None].expand(len(fb), MIX_K))
  # the layer entry point runs the same call
  layer = tfrs.layers.factorized_top_k.BruteForce(k=MIX_K).index(c)
  assert layer._tc_index is not None
  ls, li = layer(q)
  _assert_fallback(_tc_rows(ops, MIX_Q, MIX_N, MIX_D, MIX_K), MIX_FALLBACK)
  assert torch.equal(li.to(torch.int64), i) and torch.equal(_bits(ls), _bits(s))


@pytest.mark.parametrize("identifiers", ["default", "duplicated"])
def test_mixed_fallback_exclude(ops, mixed, identifiers):
  import recommenders_b200 as tfrs
  q, c, image = mixed
  Q, N, d, k, E = MIX_Q, MIX_N, MIX_D, MIX_K, MIX_E
  ids = None if identifiers == "default" else (torch.arange(N, device="cuda") // 3) * 10 + 7   # triples share an id
  cn = c.cpu().numpy()
  os_, oi = orc.topk_scan(q.cpu().numpy(), cn, k + E)       # the over-fetched exact list
  g = torch.Generator(device="cuda"); g.manual_seed(103)
  ex_rows = torch.randint(0, N, (Q, E), generator=g, device="cuda")
  oi_t = torch.from_numpy(oi).cuda()
  ex_rows[:, 0] = oi_t[:, 0]; ex_rows[:, 1] = oi_t[:, 3]; ex_rows[::3, 2] = oi_t[::3, k + E - 1]
  fb = torch.from_numpy(MIX_FALLBACK).cuda()
  ex_rows[fb, 3] = MIX_V0 + 1; ex_rows[fb, 4] = MIX_V0 + k          # hits inside the tied block
  ex_rows[fb[::2], 2] = MIX_V0 + 2 * k                              # and one below the over-fetched list
  ex = ex_rows if ids is None else ids[ex_rows]
  s, i = ops.topk_tc_exclude(q, c, image, k, ex, identifiers=ids)
  _assert_fallback(_tc_rows(ops, Q, N, d, k + E), MIX_FALLBACK)
  # the reference's rule on the oracle's exact over-fetched list
  idn = np.arange(N) if ids is None else ids.cpu().numpy()
  es_, eid = orc.exclude(os_, idn[oi], ex.cpu().numpy(), k)
  np.testing.assert_array_equal(idn[i.cpu().numpy()], eid)
  np.testing.assert_array_equal(s.cpu().numpy().view(np.uint32), es_.view(np.uint32))
  # indices: the standalone re-rank kernel on the exact CUDA-core list
  xs, xi = ops.topk_scan(q, c, k + E)
  rs, ri = ops.exclude_rerank(xs, xi, ex, k, identifiers=ids)
  assert torch.equal(i, ri) and torch.equal(_bits(s), _bits(rs))
  # from scratch on the CPU, and through the layer
  cs, ci = orc.query_with_exclusions(lambda qq, kk: (lambda r: (r[0], idn[r[1]]))(orc.topk_scan(qq, cn, kk)),
                                     q.cpu().numpy(), ex.cpu().numpy(), k)
  np.testing.assert_array_equal(idn[i.cpu().numpy()], ci)
  layer = tfrs.layers.factorized_top_k.BruteForce(k=k).index(c, ids)
  ls, lid = layer.query_with_exclusions(q, ex)
  _assert_fallback(_tc_rows(ops, Q, N, d, k + E), MIX_FALLBACK)
  np.testing.assert_array_equal(lid.cpu().numpy(), ci)
  np.testing.assert_array_equal(ls.cpu().numpy().view(np.uint32), cs.view(np.uint32))


def test_mixed_fallback_count(ops, mixed):
  q, c, image = mixed
  Q, N, d, k = MIX_Q, MIX_N, MIX_D, MIX_K
  full = orc.scores(q.cpu().numpy(), c.cpu().numpy())
  srt = -np.sort(-full, axis=1)
  pos = np.empty(Q, np.float32)
  ranks = [0, k - 2, k - 1, k, k + 1, 2 * k, 500]
  for r in range(Q):
    pos[r] = srt[r, ranks[r % len(ranks)]]
  pos[2], pos[3], pos[4] = np.nan, np.inf, -np.inf
  pos[5] = np.float32(1.5)                                           # not a candidate's score
  count_fb = []
  for j, r in enumerate(MIX_FALLBACK):
    tie = np.float32(q[r, 0].item() * MIX_A)
    if r == 7:
      pos[r] = np.inf                         # nothing above: no candidate is ambiguous, stays on the tensor cores
    elif r == 298:
      pos[r] = -np.inf                        # all listed candidates are definite: count = k on the tensor cores
    elif r == 256:
      pos[r] = np.nan
    else:                                     # inside / just above / just below the ties: the band overflows
      pos[r] = [tie, np.nextafter(tie, np.float32(np.inf)), np.nextafter(tie, np.float32(-np.inf))][j % 3]
      count_fb.append(r)
  cnt = ops.topk_tc_count(q, c, image, k, torch.from_numpy(pos).cuda())
  _assert_fallback(_tc_rows(ops, Q, N, d, k), count_fb)
  np.testing.assert_array_equal(cnt.cpu().numpy(), _count_expected(full, pos, k))


def test_mixed_fallback_factorized_topk_metric(ops, mixed):
  import recommenders_b200 as tfrs
  q, c, _ = mixed
  ks = (1, 5, 10, MIX_K)
  g = torch.Generator(device="cuda"); g.manual_seed(104)
  true = torch.randint(0, MIX_N, (MIX_Q,), generator=g, device="cuda")
  fb = torch.from_numpy(MIX_FALLBACK).cuda()
  true[fb] = MIX_V0 + fb                   # the positive of a planted row is v itself: it ties with the whole block
  layer = tfrs.layers.factorized_top_k.BruteForce().index(c)
  m = tfrs.metrics.FactorizedTopK(layer, ks=ks)
  m.update_state(q, c[true])
  _assert_fallback(_tc_rows(ops, MIX_Q, MIX_N, MIX_D, MIX_K), MIX_FALLBACK)
  cn = c.cpu().numpy()
  exp = orc.factorized_top_k_update(q.cpu().numpy(), cn[true.cpu().numpy()], lambda qq, kk: orc.topk_scan(qq, cn, kk), ks)
  for got, (num, den) in zip(m.result(), exp):
    assert abs(got - num / den) < 1e-6


# ------------------------------------------------------------------------------------------------
# 2. COUNT positives where pos +- eps straddles the filter threshold T_q and the sampled bound L_q
# ------------------------------------------------------------------------------------------------
E_REL, E_ACC = 0.00108, 0.00013   # csrc/topk_tc.cu: margin_q = 2 eps_q + E_ACC |q| |c|_max, cut_q = 2 eps_q


def test_count_positives_at_filter_threshold(ops):
  Q, N, d, k = 256, 65536, 64, 100
  c = _rand((N, d), 201); q = _rand((Q, d), 202)
  image = ops.index_build(c)
  ops.topk_tc_count(q, c, image, k, torch.zeros(Q, device="cuda"))   # T_q does not depend on the positives
  rows = _tc_rows(ops, Q, N, d, k)
  assert not rows["fallback"].any() and not rows["seg_ovf"].any()
  # screening units -> score units: 2^-(corpus exponent + row exponent), both exact powers of two.  Both exponents are
  # the library's own (index header, workspace), checked against the rescale rule restated from the inputs.
  e_c = int(image[8:12].view(torch.int32).item())
  e_q = rows["qexp"].astype(np.int64)
  assert e_c == 15 - math.frexp(float(c.abs().max()))[1]
  np.testing.assert_array_equal(e_q, [15 - math.frexp(float(a))[1] for a in q.abs().amax(1).cpu().numpy()])
  unit = np.ldexp(1.0, -(e_c + e_q))
  T = rows["thr"].astype(np.float64) * unit
  eps = 0.5 * rows["cut"].astype(np.float64) * unit
  L = T + 2 * eps * (1 + E_ACC / (2 * E_REL))
  full = orc.scores(q.cpu().numpy(), c.cpu().numpy())
  # and the converted T_q against the survivors the filter kept: |screening - exact| <= eps, so
  # #{exact >= T + eps} <= n <= #{exact >= T - eps} for every row
  full64 = full.astype(np.float64)
  assert ((full64 >= (T + eps)[:, None]).sum(1) <= rows["n"]).all()
  assert (rows["n"] <= (full64 >= (T - eps)[:, None]).sum(1)).all()
  srt = -np.sort(-full, axis=1)
  n_exact_T = (full >= T[:, None].astype(np.float32)).sum(1)     # rank of T_q among the exact scores
  pos = np.empty(Q, np.float32)
  for r in range(Q):
    kinds = [srt[r, k - 2], srt[r, k - 1], srt[r, k], srt[r, 2 * k - 1],
             srt[r, max(n_exact_T[r] - 1, 0)], srt[r, n_exact_T[r]],
             T[r], T[r] + eps[r], T[r] - eps[r], L[r], L[r] + eps[r], L[r] - eps[r],
             srt[r, np.argmin(np.abs(srt[r, :4 * k] - L[r]))]]
    pos[r] = np.float32(kinds[r % len(kinds)])
  cnt = ops.topk_tc_count(q, c, image, k, torch.from_numpy(pos).cuda())
  _assert_fallback(_tc_rows(ops, Q, N, d, k), [])
  np.testing.assert_array_equal(cnt.cpu().numpy(), _count_expected(full, pos, k))


# ------------------------------------------------------------------------------------------------
# 3. shape sweep on ordinary random data: no row may need the fallback
# ------------------------------------------------------------------------------------------------
_D = [1, 2, 8, 15, 16, 17, 63, 64, 65, 127, 128]           # 65: first shape of the SS path; residues of the 64-wide slab
_QS = [1, 63, 64, 65, 255, 256, 257]                        # either side of the 64-row warpgroup / 256-row CTA
_NK = [(20000, 10), (33333, 50), (40961, 100), (25601, 1), (50000, 32)]
_SWEEP = [(d, _QS[(j + off) % len(_QS)], *_NK[(j + off) % len(_NK)]) for j, d in enumerate(_D) for off in (0, 3)]


@pytest.mark.parametrize("d,Q,N,k", _SWEEP)
def test_shape_sweep(ops, d, Q, N, k):
  _check_topk(ops, _rand((Q, d), 1000 + d), _rand((N, d), 2000 + Q), k)


@pytest.mark.parametrize("k", [1, 31, 32, 33, 255, 256])
def test_smallest_corpus_per_k(ops, k):
  Q, d = 65, 64
  tiles = next(t for t in range(1, 1 << 12) if ops.tc_supported(Q, t * TILE, d, k))
  n_min = tiles * TILE
  assert not ops.tc_supported(Q, n_min - 1, d, k)
  for N in (n_min, n_min + 1):
    _check_topk(ops, _rand((Q, d), 3000 + k), _rand((N, d), 4000 + N), k)


@pytest.mark.parametrize("m", [150, 257])
@pytest.mark.parametrize("delta", [-1, 0, 1])
def test_tile_edges(ops, m, delta):
  _check_topk(ops, _rand((100, 64), 5000 + m), _rand((TILE * m + delta, 64), 6000 + m + delta), 50, index_offset=7)


def test_exclude_and_count_at_k_256(ops):
  Q, N, d = 100, 131072, 64
  c = _rand((N, d), 301); q = _rand((Q, d), 302)
  image = ops.index_build(c)
  qn, cn = q.cpu().numpy(), c.cpu().numpy()
  k, E = 250, 6                                                     # k + E = 256 candidates are fetched
  os_, oi = orc.topk_scan(qn, cn, k + E)
  g = torch.Generator(device="cuda"); g.manual_seed(303)
  ex = torch.randint(0, N, (Q, E), generator=g, device="cuda")
  oi_t = torch.from_numpy(oi).cuda()
  ex[:, 0] = oi_t[:, 0]; ex[:, 1] = oi_t[:, 100]; ex[:, 2] = oi_t[:, 249]; ex[::2, 3] = oi_t[::2, 255]
  s, i = ops.topk_tc_exclude(q, c, image, k, ex)
  _assert_fallback(_tc_rows(ops, Q, N, d, k + E), [])
  es_, ei_ = orc.exclude(os_, oi, ex.cpu().numpy(), k)
  np.testing.assert_array_equal(i.cpu().numpy(), ei_)
  np.testing.assert_array_equal(s.cpu().numpy().view(np.uint32), es_.view(np.uint32))
  k = 256
  full = orc.scores(qn, cn)
  srt = -np.sort(-full, axis=1)
  ranks = [0, k - 2, k - 1, k, k + 1, 300, 2 * k]
  pos = np.array([srt[r, ranks[r % len(ranks)]] for r in range(Q)], np.float32)
  pos[3], pos[4], pos[5] = np.nan, np.inf, -np.inf
  cnt = ops.topk_tc_count(q, c, image, k, torch.from_numpy(pos).cuda())
  _assert_fallback(_tc_rows(ops, Q, N, d, k), [])
  np.testing.assert_array_equal(cnt.cpu().numpy(), _count_expected(full, pos, k))


# ------------------------------------------------------------------------------------------------
# 4. the selection and threshold branches, by construction
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("N,k,extra,n_lo,n_hi,wide_bins", [
    (65536, 64, 0, 64, 512, False),        # tau from warp_kth_largest_regs<16>, tc_threshold_kernel<16>
    (131072, 128, 250, 512, 1024, False),  # warp_kth_largest_regs<32>
    (262144, 256, 476, 1024, 2048, True),  # warp_kth_largest_smem; n_bins > 512: tc_threshold_kernel<32>
])
def test_select_branches(ops, N, k, extra, n_lo, n_hi, wide_bins):
  """A plateau of M candidates scores ~1 (distinct values, spread << the band) and every other candidate <= 0.5.  One
  plateau member sits in each 64-column half of every SAMPLED tile, so every bin maximum of the sampled pass is a plateau
  score; `extra` more sit in unsampled tiles.  The filter then keeps exactly the plateau: n = M survivors per row."""
  Q, d = 40, 64
  plan = _plan(Q, N, d, k)
  assert (plan["n_bins"] > 512) == wide_bins, plan
  full_tiles = N // TILE
  sampled = np.arange(0, full_tiles, plan["stride"])   # tile(u) = u * stride
  assert len(sampled) == plan["n_sample"]
  unsampled = np.setdiff1d(np.arange(full_tiles), sampled)
  unsampled = unsampled[np.linspace(0, len(unsampled) - 1, extra).astype(np.int64)] if extra else unsampled[:0]
  members = np.concatenate([sampled * TILE + (sampled * 7) % 64, sampled * TILE + 64 + (sampled * 11) % 64,
                            unsampled * TILE + (unsampled * 13) % TILE])
  M = len(members)
  assert n_lo < M <= n_hi and M <= plan["cap_band"], (M, plan)
  rng = np.random.default_rng(k)
  cn = rng.standard_normal((N, d)).astype(np.float32)
  cn[:, 0] = rng.uniform(-0.5, 0.5, N).astype(np.float32)
  cn[members, 0] = (1.0 + rng.permutation(M) * 2.0 ** -20).astype(np.float32)
  qn = np.zeros((Q, d), np.float32)
  qn[:, 0] = 2.0 ** (np.arange(Q) % 5 - 2)
  qn[:, 1:] = 1e-5 * rng.standard_normal((Q, d - 1))
  _, _, rows = _check_topk(ops, torch.from_numpy(qn).cuda(), torch.from_numpy(cn).cuda(), k)
  assert (rows["n_bins"] > 512) == wide_bins, rows["n_bins"]     # the library's own bin count picks the threshold kernel
  np.testing.assert_array_equal(rows["n"], np.full(Q, M), err_msg="survivors per row")
  assert not rows["seg_ovf"].any() and (rows["records"] < 8192).all()


def test_record_locator_exit(ops):
  """The select kernel's 16-bit record locator holds 13 bits of record index: a row with >= 8192 octet records falls
  back.  Candidates = [1, random]; a query e0 ties every candidate at exactly 1.0, so every octet of every segment is
  recorded.  With exactly 4 tiles per corpus part a segment holds 4 tiles x 8 octets = 32 = cap_part records: full
  but not overflowed, and the row holds segs * 32 records.

  The segment count follows the SM count (one corpus part per SM for one 256-query block): 132 SMs (H100 SXM) give
  264 segments x 32 = 8448 records, which reaches the exit; 114 SMs (H100 PCIe) give 228 x 32 = 7296, which cannot, and
  the case is skipped there."""
  Q, d, k = 200, 64, 10
  parts = _plan(Q, 1 << 20, d, k)["parts"]
  N = parts * 4 * TILE
  plan = _plan(Q, N, d, k)
  if plan["segs"] * plan["cap_part"] < 8192:
    pytest.skip(f"{parts} SMs: a row holds at most {plan['segs'] * plan['cap_part']} < 8192 records, the exit is unreachable")
  assert plan["cap_part"] == 32
  c = _rand((N, d), 401); c[:, 0] = 1.0
  q = _rand((Q, d), 402); q[:, 0] = 0.0
  planted = np.array([0, 3, 63, 64, 128, 199])
  p = torch.from_numpy(planted).cuda()
  q[p] = 0.0; q[p, 0] = 1.0
  s, i, rows = _check_topk(ops, q, c, k, planted)
  assert (rows["records"][planted] == plan["segs"] * plan["cap_part"]).all() and not rows["seg_ovf"].any()
  others = np.setdiff1d(np.arange(Q), planted)
  assert (rows["records"][others] < 8192).all()
  assert torch.equal(i[p], torch.arange(k, device="cuda").expand(len(planted), k)) and bool((s[p] == 1.0).all())


# ------------------------------------------------------------------------------------------------
# 5. per-row exponent and magnitude edges, signed zero
# ------------------------------------------------------------------------------------------------
def _neg_tiny(rng, shape):
  return (-1e-25 * (1.0 + np.abs(rng.standard_normal(shape)))).astype(np.float32)


def _pos_tiny(rng, shape):
  return (1e-25 * (1.0 + np.abs(rng.standard_normal(shape)))).astype(np.float32)


@pytest.mark.parametrize("d", [64, 33])
def test_magnitude_edges_and_signed_zero(ops, d):
  """One batch: an all-zero query (its screening scores all tie: the exact fallback), rows scaled by 1e-30 and 1e+30,
  subnormal queries, and queries q ~ -1e-25 against non-negative candidates.  Those score every candidate c ~ 1e-25 at
  -0.0f (every product underflows to -0), the all-zero candidate at +0.0f and everything else below zero: their top-k is
  the zero scores in index order, with the chain's own sign bits (tensor-core rows, re-scored at d = 64 by the 8-lane
  chain and otherwise by exact_score).  The +0.0f candidate sits between -0.0f ones, so -0 must tie with +0 and rank by
  index: ranking -0 below +0 would move it to the front."""
  N, Q, k = 40000, 96, 20
  rng = np.random.default_rng(d)
  cn = np.abs(rng.standard_normal((N, d))).astype(np.float32)
  cn[3000] = 0.0                                       # the all-zero candidate, between tiny[2] and tiny[3]
  cn[100:200, : d // 2] = -0.0                         # -0.0 entries
  cn[300:310, :4] = np.float32(1e-40)                  # subnormal entries
  tiny = np.arange(977, N, 977)[:40]
  cn[tiny] = _pos_tiny(rng, (len(tiny), d))
  qn = rng.standard_normal((Q, d)).astype(np.float32)
  qn[10] = 0.0                                         # all-zero query
  qn[20] *= np.float32(1e-30); qn[21] *= np.float32(1e30)
  qn[22] = (1e-39 * rng.standard_normal(d)).astype(np.float32)   # subnormal query
  qn[40, :4] = np.float32(1e-41)                       # subnormal entries in a normal query
  neg = [30, 31, 95]
  qn[neg] = _neg_tiny(rng, (len(neg), d))
  q, c = torch.from_numpy(qn).cuda(), torch.from_numpy(cn).cuda()
  s, i, _ = _check_topk(ops, q, c, k, [10])
  zero_rows = np.sort(np.concatenate([[3000], tiny]))[:k]
  zero_bits = np.where(zero_rows == 3000, 0, 0x80000000).astype(np.uint32)
  assert zero_bits[3] == 0 and zero_bits[:3].all()
  sb = s.cpu().numpy().view(np.uint32)
  for r in neg:
    np.testing.assert_array_equal(i[r].cpu().numpy(), zero_rows)
    np.testing.assert_array_equal(sb[r], zero_bits, err_msg="the chain's -0.0f must survive the re-scoring")
  # EXCLUDE on the same batch: the tensor-core re-rank and, for the all-zero query, tc_exclude_fallback_kernel
  E = 2
  ex = torch.stack([i[:, 1], i[:, 4]], 1)
  es, ei = ops.topk_tc_exclude(q, c, ops.index_build(c), k, ex)
  _assert_fallback(_tc_rows(ops, Q, N, d, k + E), [10])
  cs, ci = orc.query_with_exclusions(lambda qq, kk: orc.topk_scan(qq, cn, kk), qn, ex.cpu().numpy(), k)
  np.testing.assert_array_equal(ei.cpu().numpy(), ci)
  np.testing.assert_array_equal(es.cpu().numpy().view(np.uint32), cs.view(np.uint32))


@pytest.mark.parametrize("d", [64, 40])
def test_signed_zero_in_fallback_rows(ops, d):
  """Queries q ~ -1e-25 against a block of 1500 candidates: 1499 with c ~ 1e-25 (score -0.0f) and, inside the block, one
  all-zero candidate (score +0.0f).  1500 exact ties at zero overflow the survivor keys, so those rows take the exact
  fallback, whose TOPK output and EXCLUDE re-rank must keep the -0.0f bits and rank the +0.0f candidate by its index
  among them.  The other queries are non-negative, so their top-k is far above the zero block (a query whose every score
  is negative would meet the same ties) and they stay on the tensor cores."""
  N, Q, k, E = 20000, 64, 20, 3
  rng = np.random.default_rng(100 + d)
  cn = np.abs(rng.standard_normal((N, d))).astype(np.float32)
  cn[4000:5500] = _pos_tiny(rng, (1500, d))
  cn[4010] = 0.0
  qn = np.abs(rng.standard_normal((Q, d))).astype(np.float32)
  neg = np.array([0, 31, 32, 63])
  qn[neg] = _neg_tiny(rng, (len(neg), d))
  q, c = torch.from_numpy(qn).cuda(), torch.from_numpy(cn).cuda()
  s, i, _ = _check_topk(ops, q, c, k, neg)
  sb = s.cpu().numpy().view(np.uint32)
  zero_rows = np.arange(4000, 4000 + k)
  zero_bits = np.where(zero_rows == 4010, 0, 0x80000000).astype(np.uint32)
  for r in neg:
    np.testing.assert_array_equal(i[r].cpu().numpy(), zero_rows)
    np.testing.assert_array_equal(sb[r], zero_bits)
  ex = torch.stack([i[:, 0], i[:, 2], i[:, k - 1]], 1)
  es, ei = ops.topk_tc_exclude(q, c, ops.index_build(c), k, ex)
  _assert_fallback(_tc_rows(ops, Q, N, d, k + E), neg)
  cs, ci = orc.query_with_exclusions(lambda qq, kk: orc.topk_scan(qq, cn, kk), qn, ex.cpu().numpy(), k)
  np.testing.assert_array_equal(ei.cpu().numpy(), ci)
  np.testing.assert_array_equal(es.cpu().numpy().view(np.uint32), cs.view(np.uint32))
  hit = ci[neg] == 4010                      # the +0.0f candidate, kept in every fallback row's list among the -0.0f ones
  assert (hit.sum(1) == 1).all() and (cs[neg].view(np.uint32)[hit] == 0).all()
