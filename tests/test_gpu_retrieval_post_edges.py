"""Edges of the per-query steps after a top-K list (csrc/topk_post.cu) and of the hard-negative loss (csrc/hardneg.cu),
against the NumPy replays in tests/retrieval_post_oracle.py.

The kernels are fed crafted lists, through `ops` and straight through the C ABI, so each one is tested apart from the
top-K scan:
  exclusion re-rank : warp layouts (4 warps per CTA up to k_fetched = 1024, 1 above), k_out edges, exclusions that
                      repeat, miss or cover the whole list, adjusted scores that collide in float32, +-0.0, identifiers,
                      and an empty [Q, 0] exclusion matrix on the layers -- ids and score bits exact
  count_above       : k around the warp width, a strided list, ties at the positive, NaN padding, non-finite positives
  hits_accumulate   : Q around the 256-thread sweep, 1 and 16 ks, unsorted and repeated ks, zero and fractional weights,
                      non-finite positives, two calls into one accumulator -- bit for bit, and FactorizedTopK on Streaming
  hard negatives    : the positive at every 32-entry ballot edge or absent, k1 up to 2048, C = k1, every column sweep
                      of the backward, underflowing coefficients, ties with the positive on both sides of it
Bars: ids, counts, hit sums and re-ranked scores exact; hard-negative loss and dq within 1e-5 of the float64 oracle's
largest magnitude, dc the same plus the spread float atomics allow; coefficients exact wherever the replay is exact."""
import ctypes
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import retrieval_post_oracle as rpo  # noqa: E402
from oracle import oracle as orc  # noqa: E402

pytestmark = pytest.mark.gpu

F32 = np.float32
EPS32 = 2.0 ** -24


@pytest.fixture(scope="module")
def ops():
  from recommenders_b200 import ops as o
  return o


@pytest.fixture(scope="module")
def ffi():
  from recommenders_b200 import _ffi
  return _ffi


def _dev(a):
  return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _int_embeddings(n, d, seed):
  """Entries in {-1, 0, 1}: scores are small integers, exact in float32 and float64, and tie often."""
  return np.random.RandomState(seed).randint(-1, 2, size=(n, d)).astype(F32)


def _canonical_pos(q, c):
  return np.array([orc.scores(q[i:i + 1], c[i:i + 1])[0, 0] for i in range(q.shape[0])], F32)


# ------------------------------------------------------------------------------------------------
# exclusion re-rank (tfrs_topk_exclude_rerank_f32)
# ------------------------------------------------------------------------------------------------
def _xr_list(Q, kf, seed, sort=True):
  """[Q, kf] scores full of float32 collisions after - 1e5 (steps of 2^-10 around 1, ulp(1e5) = 2^-7), exact
  duplicates, +0.0 and -0.0, some spread-out scores; distinct int64 indices above 2^32 in every row."""
  rs = np.random.RandomState(seed)
  s = F32(1.0) + rs.randint(0, 64, size=(Q, kf)).astype(F32) * F32(2.0 ** -10)
  far = rs.rand(Q, kf) < 0.2
  s[far] = rs.normal(size=int(far.sum())).astype(F32) * F32(50.0)
  zero = rs.rand(Q, kf) < 0.1
  s[zero] = np.where(rs.rand(int(zero.sum())) < 0.5, F32(0.0), F32(-0.0))
  if sort:
    s = -np.sort(-s, 1)     # negating twice keeps the sign of every zero
  idx = (((np.arange(kf)[None, :] * 40503 + np.arange(Q)[:, None] * 7) % 65536).astype(np.int64) << 24) + 3
  return s, idx


def _xr_exclusions(idx, n_excl, seed):
  """n_excl = 1: a listed index on even rows, a miss on odd rows.  n_excl = 33: listed indices with repeats and misses;
  on every 4th row, when the list is that short, every listed index (the whole list is excluded)."""
  rs = np.random.RandomState(seed)
  Q, kf = idx.shape
  if n_excl == 0:
    return np.zeros((Q, 0), np.int64)
  pick = np.take_along_axis(idx, rs.randint(0, kf, size=(Q, n_excl)), 1)
  miss = rs.randint(1, 1 << 20, size=(Q, n_excl)).astype(np.int64) << 40
  if n_excl == 1:
    return np.where((np.arange(Q) % 2 == 0)[:, None], pick, miss)
  ex = np.where(rs.rand(Q, n_excl) < 0.6, pick, miss)
  ex[:, 1] = ex[:, 0]                                          # a duplicate exclusion
  if kf <= n_excl:
    ex[3::4] = np.tile(idx[3::4], (1, -(-n_excl // kf)))[:, :n_excl]
  return ex


def _xr_check(ops, s, idx, ex, k, ident=None):
  gs, gi = ops.exclude_rerank(_dev(s), _dev(idx), _dev(ex), k, identifiers=None if ident is None else _dev(ident))
  es, ei = rpo.exclude_rerank(s, idx, ex, k, identifiers=ident)
  np.testing.assert_array_equal(gi.cpu().numpy(), ei)
  np.testing.assert_array_equal(gs.cpu().numpy().view(np.uint32), es.view(np.uint32))


@pytest.mark.parametrize("Q", [1, 3, 4, 5, 4097])
@pytest.mark.parametrize("kf", [1, 31, 32, 33, 1024, 1025, 4096])
def test_exclude_rerank_warp_layouts_and_k_out(ops, kf, Q):
  s, idx = _xr_list(Q, kf, 7 * kf + Q)
  ds, di = _dev(s), _dev(idx)
  for n_excl in (0, 1, 33):
    ex = _xr_exclusions(idx, n_excl, kf + Q + n_excl)
    de = _dev(ex)
    es, ei = rpo.exclude_rerank(s, idx, ex, kf)      # every k_out below is a prefix of the full order
    for k in sorted({1, max(kf - 1, 1), kf}):
      gs, gi = ops.exclude_rerank(ds, di, de, k)
      np.testing.assert_array_equal(gi.cpu().numpy(), ei[:, :k], err_msg=f"n_excl={n_excl} k={k}")
      np.testing.assert_array_equal(gs.cpu().numpy().view(np.uint32), es[:, :k].view(np.uint32))


def test_exclude_rerank_collisions_and_signed_zeros_abi(ffi):
  """Unsorted crafted lists through the C ABI: a lower-scored entry at a LOWER position collides with a higher-scored
  one after - 1e5, so only the position rule orders them; -0.0 ahead of +0.0 ranks first (they tie after + 0)."""
  a, b = F32(1.0), F32(1.0) + F32(2.0 ** -9)
  assert a - F32(1e5) == b - F32(1e5) and a != b
  s = np.array([[a, b, F32(-0.0), F32(0.0), F32(5.0), F32(-3.0)],
                [F32(0.0), F32(-0.0), b, a, F32(-0.0), F32(1e5)],
                [b, a, F32(-0.0), F32(0.0), F32(0.0), F32(-0.0)]], F32)
  idx = np.array([[10, 11, 12, 13, 14, 15], [20, 21, 22, 23, 24, 25], [30, 31, 32, 33, 34, 35]], np.int64)
  ex = np.array([[10, 11, 99], [22, 23, 25], [30, 31, 31]], np.int64)
  out_s = torch.empty((3, 6), dtype=torch.float32, device="cuda")
  out_i = torch.empty((3, 6), dtype=torch.int64, device="cuda")
  ds, di, de = _dev(s), _dev(idx), _dev(ex)
  ffi.check(ffi.lib().tfrs_topk_exclude_rerank_f32(ffi.ptr(ds), ffi.ptr(di), 3, 6, None, ffi.ptr(de), 3, 6,
                                                   ffi.ptr(out_s), ffi.ptr(out_i), ffi.stream()), "exclude_rerank")
  es, ei = rpo.exclude_rerank(s, idx, ex, 6)
  assert ei.tolist() == [[14, 12, 13, 15, 10, 11], [20, 21, 24, 25, 22, 23], [32, 33, 34, 35, 30, 31]]
  np.testing.assert_array_equal(out_i.cpu().numpy(), ei)
  np.testing.assert_array_equal(out_s.cpu().numpy().view(np.uint32), es.view(np.uint32))


@pytest.mark.parametrize("kf,k", [(40, 10), (40, 40), (1025, 1000), (4096, 4096)])
def test_exclude_rerank_identifiers_all_and_most_excluded(ops, kf, k):
  """identifiers= path: identifiers repeat (index % 5), so one exclusion removes many entries; rows exclude nothing,
  all but one identifier (fewer entries left than k), or every identifier (the whole list, original scores kept)."""
  Q = 9
  s, idx = _xr_list(Q, kf, kf + k, sort=(kf != 40))
  idx = idx >> 24                                            # indices into the identifier table
  ident = (np.arange(65536, dtype=np.int64) % 5) * (1 << 35) + 1
  ex = np.full((Q, 6), 7, np.int64)                          # 7 is not an identifier: a miss
  ex[1::3, :4] = ident[:4]
  ex[2::3, :5] = ident[[4, 0, 3, 1, 2]]
  ex[2::3, 5] = ident[0]
  _xr_check(ops, s, idx, ex, k, ident=ident)


@pytest.mark.parametrize("N,k", [(3000, 10), (40000, 64)])
@pytest.mark.parametrize("ids", [False, True])
def test_query_with_exclusions_empty_exclusions_is_topk(ops, N, k, ids):
  """An empty [Q, 0] exclusion matrix: query_with_exclusions returns exactly the plain top-k, on BruteForce and on
  Streaming."""
  import recommenders_b200 as tfrs
  d, Q = 32, 37
  g = torch.Generator(device="cuda"); g.manual_seed(N + k)
  c = torch.randn((N, d), generator=g, device="cuda"); q = torch.randn((Q, d), generator=g, device="cuda")
  ident = (torch.arange(N, device="cuda", dtype=torch.int64) * 3 + (1 << 33)) if ids else None
  empty = torch.zeros((Q, 0), dtype=torch.int64, device="cuda")
  es, ei = ops.topk(q, c, k)
  eid = (ident[ei] if ids else ei.to(torch.int32)).cpu().numpy()
  bf = tfrs.layers.factorized_top_k.BruteForce(k=k).index(c, ident)
  ds = tfrs.data.Dataset.from_tensor_slices((ident, c) if ids else c).batch(1000)
  st = tfrs.layers.factorized_top_k.Streaming(k=k).index_from_dataset(ds)
  for layer in (bf, st):
    s, i = layer.query_with_exclusions(q, empty)
    np.testing.assert_array_equal(i.cpu().numpy(), eid)
    np.testing.assert_array_equal(s.cpu().numpy().view(np.uint32), es.cpu().numpy().view(np.uint32))


# ------------------------------------------------------------------------------------------------
# in-top-K count (tfrs_count_above_f32)
# ------------------------------------------------------------------------------------------------
def _count_case(Q, k, seed):
  """Integer scores with many ties at the positive; NaN padding at the tail of some rows; +inf, -inf and NaN
  positives; positives taken from the list itself."""
  rs = np.random.RandomState(seed)
  s = -np.sort(-rs.randint(-4, 5, size=(Q, k)).astype(F32), 1)
  pos = rs.randint(-4, 5, size=Q).astype(F32)
  if k:
    pos[::4] = s[::4, rs.randint(0, k)]
    for r in range(1, Q, 5):
      s[r, rs.randint(0, k):] = np.nan
  pos[1::7] = np.inf; pos[2::7] = -np.inf; pos[3::7] = np.nan
  return s, pos


@pytest.mark.parametrize("k", [0, 1, 31, 32, 33, 100])
def test_count_above_edges(ops, ffi, k):
  Q, ld = 37, k + 7
  s, pos = _count_case(Q, k, 100 + k)
  exp = rpo.count_above(s, pos)
  got = ops.count_above(_dev(s), _dev(pos))
  np.testing.assert_array_equal(got.cpu().numpy(), exp)
  # a strided [Q, k] view of a [Q, k + 7] buffer whose extra columns would all count
  full = np.full((Q, ld), np.inf, F32); full[:, :k] = s
  dfull, dpos = _dev(full), _dev(pos)
  np.testing.assert_array_equal(ops.count_above(dfull[:, :k], dpos).cpu().numpy(), exp)
  out = torch.full((Q,), -1, dtype=torch.int32, device="cuda")
  ffi.check(ffi.lib().tfrs_count_above_f32(ffi.ptr(dfull), ld, k, ffi.ptr(dpos), Q, ffi.ptr(out), ffi.stream()),
            "count_above")
  np.testing.assert_array_equal(out.cpu().numpy(), exp)


def test_empty_batch_counts_and_sums_nothing(ops):
  """Q = 0 (torch's empty tensors have NULL data pointers): no counts, and the accumulator is left as it was."""
  cnt = ops.count_above(torch.empty((0, 10), device="cuda"), torch.empty((0,), device="cuda"))
  assert cnt.shape == (0,)
  acc = torch.tensor([1.5, 2.5, 4.0], dtype=torch.float64, device="cuda")
  ops.hits_accumulate(cnt, torch.empty((0,), device="cuda"), torch.empty((0,), device="cuda"), (1, 5), acc)
  assert acc.cpu().tolist() == [1.5, 2.5, 4.0]


def test_count_above_ties_count_as_hits(ops):
  """tf.math.in_top_k: only scores strictly above the positive push it down."""
  s = np.array([[3, 2, 2, 2, 1], [2, 2, 2, 2, 2], [5, 4, 3, 2, 1]], F32)
  pos = np.array([2, 2, 0.5], F32)
  assert ops.count_above(_dev(s), _dev(pos)).cpu().numpy().tolist() == [1, 0, 5]


# ------------------------------------------------------------------------------------------------
# hit sums (tfrs_topk_hits_accumulate)
# ------------------------------------------------------------------------------------------------
KS_SETS = {"one": (5,), "sixteen": tuple(range(1, 161, 10)), "unsorted_repeated": (10, 1, 100, 5, 5, 1, 50)}


@pytest.mark.parametrize("ks_name", sorted(KS_SETS))
@pytest.mark.parametrize("Q", [1, 255, 256, 257, (1 << 20) + 1])
def test_hits_accumulate_bitwise(ops, Q, ks_name):
  ks = KS_SETS[ks_name]
  rs = np.random.RandomState(Q % 1000 + len(ks))
  acc0 = np.array(rs.normal(size=len(ks) + 1) * 10.0)
  acc = _dev(acc0)
  exp = acc0
  for call, weights in enumerate(("none", "zero", "fractional")):
    cnt = rs.randint(0, 120, size=Q).astype(np.int32)
    cnt[::11] = 1 << 30                                       # "not retrieved" (the identifier branch)
    pos = rs.normal(size=Q).astype(F32)
    pos[::13] = np.inf; pos[5::13] = -np.inf; pos[7::13] = np.nan
    w = {"none": None, "zero": np.zeros(Q, F32),
         "fractional": (rs.rand(Q) * 3.0 - 0.5).astype(F32)}[weights]
    if w is not None and Q > 3:
      w[2::17] = 0.0
    ops.hits_accumulate(_dev(cnt), _dev(pos), None if w is None else _dev(w), ks, acc)
    exp = rpo.hits_accumulate(cnt, pos, w, ks, exp)          # the same accumulator, call after call
    np.testing.assert_array_equal(acc.cpu().numpy().view(np.uint64), exp.view(np.uint64), err_msg=f"call {call}")


def test_factorized_top_k_on_streaming_exact_ratios():
  """FactorizedTopK on a Streaming layer (the list-based count and the hit sums, two weighted updates) gives every
  ratio exactly; integer embeddings put many corpus scores level with the positive."""
  import recommenders_b200 as tfrs
  N, d, ks = 5000, 8, (1, 5, 10, 50, 100)
  c = _int_embeddings(N, d, 21)
  ds = tfrs.data.Dataset.from_tensor_slices(_dev(c)).batch(512)
  metric = tfrs.metrics.FactorizedTopK(tfrs.layers.factorized_top_k.Streaming(k=max(ks)).index_from_dataset(ds), ks=ks)
  acc = None
  for step, Q in enumerate((300, 257)):
    rs = np.random.RandomState(22 + step)
    q = _int_embeddings(Q, d, 23 + step)
    true = c[rs.randint(0, N, Q)]
    w = (rs.rand(Q) * 2).astype(F32)
    metric.update_state(_dev(q), _dev(true), sample_weight=_dev(w))
    pos = _canonical_pos(q, true)
    top_s, _ = orc.topk_scan(q, c, max(ks))
    cnt = rpo.count_above(top_s, pos)
    assert ((cnt < 100) & (top_s[np.arange(Q), np.minimum(cnt, 99)] == pos)).any()   # ties at the positive
    acc = rpo.hits_accumulate(cnt, pos, w, ks, acc)
  assert metric.result() == [a / acc[-1] for a in acc[:-1]]


# ------------------------------------------------------------------------------------------------
# hard-negative loss (tfrs_hardneg_loss_fwd / _bwd)
# ------------------------------------------------------------------------------------------------
POS_SLOTS = (0, 31, 32, 33, -1, None)     # list position of the positive (-1 = k1 - 1, None = not in the list)


def _hn_list(B, k1, C, temp, seed, ties=False):
  """Crafted [B, k1] lists (scores descending, distinct candidate ids < C).  Row r holds its positive at
  POS_SLOTS[r % 6] when that position exists, else not at all.  At T = 0.05 the tail of every list lies 12 below the
  head, so those coefficients underflow to exactly 0.  `ties`: the positive's score is shared by its neighbours."""
  rs = np.random.RandomState(seed)
  top_s = -np.sort(-rs.normal(size=(B, k1)).astype(F32), 1) * F32(0.5)
  if temp == 0.05:
    top_s[:, k1 // 2:] -= F32(12.0)
  top_i = np.empty((B, k1), np.int64)
  pos = np.empty(B, F32)
  for r in range(B):
    slot = POS_SLOTS[r % len(POS_SLOTS)]
    p = None if slot is None else (k1 - 1 if slot == -1 else slot)
    if p is not None and p >= k1:
      p = None
    others = rs.permutation(np.delete(np.arange(C), r))
    if p is None and others.shape[0] < k1:
      p = rs.randint(k1)                                       # C = k1: every candidate, the positive too, is listed
    top_i[r] = others[:k1] if p is None else np.insert(others[:k1 - 1], p, r)
    if p is not None:
      if ties:
        top_s[r, max(p - 2, 0):p + 3] = top_s[r, p]
      pos[r] = top_s[r, p]
    else:
      pos[r] = top_s[r, -1] - F32(0.25) if not ties else top_s[r, -1]
  return top_s, top_i, pos


def _hn_fwd(ffi, top_s, top_i, pos, inv_t, w):
  B, k1 = top_s.shape
  loss = torch.empty((1,), dtype=torch.float32, device="cuda")
  coef = torch.empty((B, k1 + 2), dtype=torch.float32, device="cuda")
  ds, di, dp = _dev(top_s), _dev(top_i), _dev(pos)
  dw = None if w is None else _dev(w)
  ffi.check(ffi.lib().tfrs_hardneg_loss_fwd(ffi.ptr(ds), ffi.ptr(di), B, k1, ffi.ptr(dp), ctypes.c_float(inv_t),
                                            ffi.ptr(dw), ffi.ptr(loss), ffi.ptr(coef), ffi.stream()), "hardneg_loss_fwd")
  return float(loss), coef.cpu().numpy()


def _hn_bwd(ffi, q, c, top_i, coef, grad_loss=None):
  B, d = q.shape
  C = c.shape[0]
  dq = torch.full((B, d), np.nan, dtype=torch.float32, device="cuda")
  dc = torch.full((C, d), np.nan, dtype=torch.float32, device="cuda")
  dq_, dc_, di, dcoef = _dev(q), _dev(c), _dev(top_i), _dev(coef.astype(F32))
  g = None if grad_loss is None else torch.tensor([grad_loss], dtype=torch.float32, device="cuda")
  ffi.check(ffi.lib().tfrs_hardneg_loss_bwd(ffi.ptr(dq_), ffi.ptr(dc_), B, C, d, ffi.ptr(di), top_i.shape[1],
                                            ffi.ptr(dcoef), ffi.ptr(g), ffi.ptr(dq), ffi.ptr(dc), ffi.stream()),
            "hardneg_loss_bwd")
  return dq.cpu().numpy(), dc.cpu().numpy()


def _within(got, ref, rel, what, extra=0.0):
  ref = np.asarray(ref, np.float64)
  err = np.abs(np.asarray(got, np.float64) - ref)
  bar = rel * np.abs(ref).max() + extra
  assert np.all(err <= bar), f"{what}: max err {err.max():.3e}, bar {np.max(bar):.3e}"


def _loss_within(got, ref, w_sum):
  # every row loss is >= 0; float32 log of a sum near 1 is off by ~2^-24 per unit weight, hence the w_sum floor
  assert abs(got - ref) <= 1e-5 * max(abs(ref), w_sum), (got, ref)


def _check_coefficients(coef, top_s, top_i, pos, inv_t, w):
  ref = rpo.hardneg_coefficients(top_s, top_i, pos, inv_t, w)
  B, k1 = top_s.shape
  # a coefficient is w/T times a probability (minus 1 for the positive): float32 is exact to ~2^-24 of w/T, however
  # small the probability, so the bar is 1e-5 of the largest w/T
  scale = float(F32(inv_t)) * (1.0 if w is None else float(np.max(w)))
  _within(coef[:, :k1 + 1], ref[:, :k1 + 1], 1e-5, "coefficients", extra=1e-5 * scale)
  drop = rpo.hardneg_drop(top_i)
  assert np.all(coef[np.arange(B), drop] == 0.0), "the dropped entry must have a zero coefficient"
  deep = ref[:, :k1] < 1e-60                                  # far below the smallest float32: exactly 0 on the GPU
  assert np.all(coef[:, :k1][deep] == 0.0)
  return ref


@pytest.mark.parametrize("temp", [0.05, 1.0, 20.0])
@pytest.mark.parametrize("B", [1, 7, 8, 9, 257])
@pytest.mark.parametrize("k1", [2, 32, 33, 64, 2048])
def test_hardneg_forward_crafted_lists(ffi, k1, B, temp):
  C = max(B, k1) if B % 2 else max(B, k1) + 5                  # C = k1 whenever B <= k1 and B is odd
  top_s, top_i, pos = _hn_list(B, k1, C, temp, 1000 * k1 + B)
  inv_t = 1.0 / temp
  for w in (None, np.where(np.arange(B) % 3 == 1, 0.0, np.random.RandomState(B).rand(B) + 0.3).astype(F32)):
    loss, coef = _hn_fwd(ffi, top_s, top_i, pos, inv_t, w)
    ref = _check_coefficients(coef, top_s, top_i, pos, inv_t, w)
    if w is not None:
      assert np.all(coef[w == 0.0] == 0.0)                   # zero weight: no loss, no gradient
    if temp == 0.05:                                          # the underflow edge is reached (not on dropped entries)
      kept = np.ones((B, k1), bool); kept[np.arange(B), rpo.hardneg_drop(top_i)] = False
      assert ((ref[:, :k1] < 1e-60) & kept).any()
    _loss_within(loss, ref[:, k1 + 1].sum(), B if w is None else float(w.sum()))


@pytest.mark.parametrize("k1", [2, 33, 64])
def test_hardneg_forward_ties_with_the_positive(ffi, k1):
  """Neighbours of the positive share its score: only the id decides what is dropped.  With every score equal to 0 the
  float32 coefficients are exact: w/T / z for kept entries, (1/z - 1) w/T for the positive, 0 for the dropped entry."""
  B = 13
  top_s, top_i, pos = _hn_list(B, k1, 2 * k1 + B, 1.0, k1, ties=True)
  loss, coef = _hn_fwd(ffi, top_s, top_i, pos, 1.0, None)
  ref = _check_coefficients(coef, top_s, top_i, pos, 1.0, None)
  _loss_within(loss, ref[:, k1 + 1].sum(), B)
  w = np.random.RandomState(k1).rand(B).astype(F32) + F32(0.5)
  inv_t = F32(1.0 / 0.05)
  zs, zp = np.zeros_like(top_s), np.zeros_like(pos)
  _, coef = _hn_fwd(ffi, zs, top_i, zp, float(inv_t), w)
  z = F32(k1)                                                  # k1 - 1 kept entries + the positive, each exp(0) = 1
  g = w * inv_t / z
  exp = np.repeat(g[:, None], k1, 1)
  exp[np.arange(B), rpo.hardneg_drop(top_i)] = 0.0
  np.testing.assert_array_equal(coef[:, :k1].view(np.uint32), exp.view(np.uint32))
  np.testing.assert_array_equal(coef[:, k1].view(np.uint32), ((F32(1.0) / z - F32(1.0)) * w * inv_t).view(np.uint32))


@pytest.mark.parametrize("d", [1, 31, 32, 33, 64, 65, 129])
@pytest.mark.parametrize("B", [1, 7, 8, 9, 257])
def test_hardneg_backward_column_sweeps(ffi, B, d):
  """The backward alone, fed float32 coefficients: dq (fixed order) and dc (atomics) against float64 on the same
  coefficients, including exact zeros (skipped) and a list whose candidates repeat across rows."""
  k1, C = 33, B + 40
  rs = np.random.RandomState(B * 1000 + d)
  top_s, top_i, pos = _hn_list(B, k1, C, 0.05, d)
  coef = rpo.hardneg_coefficients(top_s, top_i, pos, 20.0, None).astype(F32)
  assert (coef[:, :k1] == 0).sum() > B                      # the dropped entries and the underflowed tail
  q = rs.normal(size=(B, d)).astype(F32); c = rs.normal(size=(C, d)).astype(F32)
  for g in (None, 0.75):
    dq, dc = _hn_bwd(ffi, q, c, top_i, coef, g)
    rdq, rdc, rabs, n = rpo.hardneg_grads(q, c, top_i, coef, 1.0 if g is None else g)
    _within(dq, rdq, 1e-5, "dq")
    _within(dc, rdc, 1e-5, "dc", extra=n[:, None] * EPS32 * rabs)
    untouched = n == 0
    assert np.all(dc[untouched] == 0.0)                     # dc is zeroed by the call


def _tie_rows(q, c, k1):
  """Per row: the raw top-k1 list (score desc, index asc) leaves out the positive because lower-index ties fill it
  ("lower"), or holds the positive and cuts a higher-index tie ("higher")."""
  s = orc.scores(q, c)
  _, top_i = orc.topk_scan(q, c, k1)
  out = {"lower": [], "higher": []}
  for i in range(q.shape[0]):
    tie = np.flatnonzero(s[i] == s[i, i])
    listed = set(top_i[i].tolist())
    if i not in listed and any(j < i and j in listed for j in tie):
      out["lower"].append(i)
    if i in listed and any(j > i and j not in listed for j in tie):
      out["higher"].append(i)
  return out


@pytest.mark.parametrize("pattern,B,C,d,n,temp", [("lower", 257, 400, 6, 20, None), ("higher", 9, 40, 4, 10, 0.05),
                                                   ("both", 64, 100, 7, 30, 20.0), ("all", 257, 2048, 12, 2047, 1.0)])
def test_retrieval_task_hard_negative_ties(ops, monkeypatch, pattern, B, C, d, n, temp):
  """tasks.Retrieval(num_hard_negatives=n) end to end on integer embeddings with duplicated candidate rows: score ties
  with the positive sit at the n + 1 boundary on the side the case names, and the loss and both gradients match the
  float64 oracle (lower index first among ties, positive always kept).  "all": k1 = C = 2048, every candidate is
  listed, duplicates included."""
  import recommenders_b200 as tfrs
  q = _int_embeddings(B, d, B + n); c = _int_embeddings(C, d, C + n)
  for i in range(2, B, 3):
    if pattern in ("lower", "both", "all"):
      c[i - 1] = c[i]
    if pattern in ("higher", "both", "all"):
      c[min(i + B, C - 1)] = c[i]
  k1 = min(n + 1, C)
  rows = _tie_rows(q, c, k1)
  for side in {"lower": ("lower",), "higher": ("higher",), "both": ("lower", "higher"), "all": ()}[pattern]:
    assert rows[side], f"no row reaches the '{side}' tie edge"
  w = np.random.RandomState(n).rand(B).astype(F32)
  w[::5] = 0.0
  monkeypatch.setattr(ops, "scores", lambda *a, **k: (_ for _ in ()).throw(AssertionError("logits were materialised")))
  qg = _dev(q).requires_grad_(True); cg = _dev(c).requires_grad_(True)
  task = tfrs.tasks.Retrieval(num_hard_negatives=n, temperature=temp)
  loss = task(qg, cg, sample_weight=_dev(w), compute_metrics=False)
  loss.backward()
  rl, rdq, rdc = orc.retrieval_loss_and_grads_general(q, c, w, temp, num_hard_negatives=n)
  _loss_within(float(loss.detach()), rl, float(w.sum()))
  _within(qg.grad.cpu().numpy(), rdq, 1e-5, "dq")
  top_s, top_i = orc.topk_scan(q, c, k1)
  coef = rpo.hardneg_coefficients(top_s, top_i, _canonical_pos(q, c[:B]), 1.0 if temp is None else 1.0 / temp, w)
  _, _, rabs, cnt = rpo.hardneg_grads(q, c, top_i, coef)
  _within(cg.grad.cpu().numpy(), rdc, 1e-5, "dc", extra=cnt[:, None] * EPS32 * rabs)
