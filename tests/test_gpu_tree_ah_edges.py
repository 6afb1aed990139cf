"""Edge grid of TreeAH (K9, csrc/tree_ah.cu): every block width and code-word count of the build and the int8 LUT, every
slice count and merge route of the search, the k / k' / probe caps, empty and tiny leaves, and the build kernels on
adversarial inputs -- all bit for bit against tests/tree_ah_oracle.py.  Run with -m gpu.

The slice count, the query chunk and the merge route are restated in tree_ah_oracle.py (`slices`, `query_chunk`,
`tree_merge`); `test_the_plan_mirror_matches_the_search_workspace` holds the restatement to the kernel's own plan and
`test_the_grid_reaches_every_edge` shows that the cases below land on each side of every limit."""
import functools
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import tree_ah_oracle as tao  # noqa: E402

pytestmark = pytest.mark.gpu

INDEX_KEYS = ("centroids", "leaf_offsets", "order", "codebooks", "codes")
F32 = np.float32


def cu(a):
  return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _np(t):
  return t.cpu().numpy()


def _same(got_s, got_i, exp_s, exp_i):
  np.testing.assert_array_equal(_np(got_i), exp_i)
  assert _np(got_s).tobytes() == np.ascontiguousarray(exp_s, F32).tobytes()


def _sms():
  return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


def _normal(N, d, seed):
  return np.random.default_rng(seed).normal(size=(N, d)).astype(F32)


def _skewed():
  """20000 rows, L = 3, no Lloyd steps: the build seeds leaf l with row perm[l], so leaf 0 takes the cluster at +10 e0,
  leaf 1 the 10 rows at -10 e0 and leaf 2, seeded with a copy of perm[0]'s row, loses every tie and stays empty."""
  N = 20000
  perm = np.random.default_rng(0).permutation(N)
  x = _normal(N, 8, 31) * F32(0.1)
  x[:, 0] += 10
  x[perm[1:12], 0] -= 20
  x[perm[2]] = x[perm[0]]
  return x


def _repeated():
  """5 distinct vectors repeated 3000 times in all over 64 leaves: duplicate centroids, so most leaves stay empty."""
  base = _normal(5, 8, 32)
  return base[np.random.default_rng(33).integers(0, 5, 3000)]


# name: (N, d, L, training_iterations, dimensions per block, corpus)
CORPORA = {
    "one_leaf": (20000, 8, 1, 2, 2, lambda: _normal(20000, 8, 41)),      # 78 slices of 256 rows -> S up to 64
    "two_leaves": (1200, 8, 2, 2, 2, lambda: _normal(1200, 8, 42)),      # S = 2
    "five_leaves": (17000, 8, 5, 2, 2, lambda: _normal(17000, 8, 43)),   # S = 13: 5 probes make 65 lists
    "skewed": (20000, 8, 3, 0, 2, _skewed),                              # S = 26 over leaves of 19990, 10 and 0 rows
    "tiny_leaves": (4096, 8, 2048, 1, 2, lambda: _normal(4096, 8, 44)),  # 2048 probes
    "many_leaves": (20000, 8, 128, 2, 2, lambda: _normal(20000, 8, 45)),
    "repeated": (3000, 8, 64, 3, 2, _repeated),
    "wide": (2000, 256, 2, 2, 1, lambda: _normal(2000, 256, 46)),        # W = 32
}


class Index:
  """One corpus built by the oracle and by ops.tree_ah_build."""

  def __init__(self, x, L, iters, dpb):
    from recommenders_b200 import ops
    self.x, self.L, self.dpb = x, L, dpb
    self.ref = tao.build(x, L, iters, dpb)
    self.gpu = ops.tree_ah_build(cu(x), L, iters, dpb)
    self.rows = cu(x)

  def check_build(self):
    for key in INDEX_KEYS:
      got, exp = _np(self.gpu[key]), np.ascontiguousarray(self.ref[key])
      assert got.shape == exp.shape and got.tobytes() == exp.tobytes(), key

  def search(self, q, P, k, kp, reorder):
    """Both sides at (P, k, k'); without reordering k' must be k, as the layer passes it."""
    from recommenders_b200 import ops
    assert reorder or kp == k
    s, i = ops.tree_ah_search(cu(q), self.gpu, self.rows if reorder else None, P, k, kp)
    es, ei = tao.search(self.ref, self.x, q, k, P, self.dpb, kp if reorder else None)
    _same(s, i, es, ei)
    return es, ei


@pytest.fixture(scope="module")
def corpus():
  @functools.lru_cache(maxsize=None)
  def get(name):
    N, d, L, iters, dpb, make = CORPORA[name]
    x = make()
    assert x.shape == (N, d)
    return Index(x, L, iters, dpb)
  return get


# ---- 1. search grid: every dimensions_per_block, code-word count and last-block width ----------------------------------
# (d, dpb): for every dpb each last-block width 1..dpb once, d from {1, 7, 63, 65, 128, 255, 256} where one has that
# width; W = ceil(ceil(d / dpb) / 8) runs from 1 to 32
WIDTHS = [(1, 1), (65, 1), (255, 1), (256, 1),
          (65, 2), (128, 2),
          (256, 3), (65, 3), (63, 3),
          (65, 4), (254, 4), (255, 4), (128, 4),
          (256, 5), (7, 5), (128, 5), (254, 5), (255, 5),
          (7, 6), (128, 6), (63, 6), (256, 6), (65, 6), (252, 6),
          (1, 7), (65, 7), (255, 7), (256, 7), (250, 7), (251, 7), (63, 7),
          (65, 8), (250, 8), (251, 8), (252, 8), (253, 8), (254, 8), (255, 8), (256, 8)]
HALF_TIES = (1.5, 2.5, -3.5, 126.5)


def _layout(d, dpb):
  """(B, W, width of the last block)."""
  B = -(-d // dpb)
  return B, (B + 7) // 8, d - (B - 1) * dpb


@pytest.mark.parametrize("d,dpb", WIDTHS)
def test_build_and_search_at_every_block_width(d, dpb):
  """Build parity (the codebooks, codes and their packing at this B and W), then the search without reordering, where a
  score is dot + s * sum(LUT), so every int8 LUT entry and the scale show in the bits, and with reordering.  The queries
  are random, zero (s = 0) and built so that T / s is exactly 1.5, 2.5, -3.5 or 126.5 (round half to even)."""
  ix = Index(_normal(1000, d, 1000 * dpb + d), 4, 2, dpb)
  ix.check_build()
  q = [_normal(4, d, d + dpb), np.zeros((1, d), F32)]
  ties = [tao.half_tie_query(ix.ref["codebooks"], d, dpb, t) for t in HALF_TIES]
  ties = [t for t in ties if t is not None]
  if ix.ref["codebooks"].shape[0] > 1:
    assert len(ties) >= 3, "the codebooks give too few exact half-integer queries"
  q = np.concatenate(q + [t[None] for t in ties])
  T, s = tao.table(q, ix.ref["codebooks"], dpb)
  assert s[4] == 0 and all(np.any(T[5 + r] % 1 == 0.5) for r in range(len(ties)))
  ix.search(q, 2, 64, 64, False)
  ix.search(q, 2, 16, 128, True)


# ---- 2. slices, merge routes, caps and padding ------------------------------------------------------------------------
# (corpus, Q, probes, k, k', reorder)
SEARCH_CASES = [
    ("one_leaf", 1, 1, 10, 10, False),         # S = 64: 64 lists, tree merge
    ("one_leaf", 1, 1, 106, 106, False),       # 64 lists x 106: region * 24 = 162,816 B, tree merge
    ("one_leaf", 1, 1, 107, 107, False),       # 64 lists x 107: 164,352 B, sorting merge
    ("one_leaf", 1, 1, 10, 106, True),
    ("one_leaf", 1, 1, 10, 107, True),
    ("one_leaf", 3, 1, 20, 60, True),          # S = min(ceil(2 SMs / 3), 78) capped at 64
    ("one_leaf", 5, 1, 20, 20, False),         # S = ceil(2 SMs / 5), interior
    ("one_leaf", 1, 1, 2048, 2048, False),     # k = 2048 without reordering
    ("two_leaves", 1, 1, 30, 30, False),       # S = 2
    ("two_leaves", 1, 2, 1706, 1706, False),   # 4 lists x 1706: 163,776 B, tree merge; k > the 1200 probed rows
    ("two_leaves", 1, 2, 1707, 1707, False),   # 163,872 B, sorting merge
    ("two_leaves", 2, 2, 1500, 1706, True),    # k and k' > the probed rows, reordered
    ("five_leaves", 1, 5, 10, 10, False),      # S = 13: 65 lists, sorting merge
    ("five_leaves", 1, 5, 10, 50, True),
    ("five_leaves", 2, 4, 10, 10, False),      # 52 lists, tree merge
    ("skewed", 1, 3, 20, 20, False),           # S = 26: slices of 0 rows in leaves 1 and 2
    ("skewed", 1, 3, 20, 40, True),
    ("skewed", 2, 1, 20, 20, False),           # query 0 probes the 10-row leaf alone: (NaN, 0) padding
    ("skewed", 2, 1, 20, 30, True),
    ("tiny_leaves", 2, 2048, 2048, 2048, False),  # k = k' = probes = 2048, S = 1, 2048 lists
    ("tiny_leaves", 2, 2048, 1, 2048, True),      # k = 1, k' = 2048
    ("many_leaves", 500, 100, 10, 2048, True),    # 100 probes x 2048: uneven query chunks
    ("wide", 2, 2, 1, 2048, True),             # W = 32 and k' = 2048: the largest AH rowselect, 53,248 B
    ("wide", 2, 2, 2048, 2048, False),         # k = 2048 over 2000 rows without reordering
    ("repeated", 3, 10, 20, 20, False),        # duplicate centroids: the probes reach empty leaves
    ("repeated", 3, 10, 20, 100, True),
]


def _queries(name, Q, d):
  q = _normal(Q, d, Q * 7 + d)
  if name == "skewed":
    q[0, 0] = -1.0   # toward the 10-row leaf
  return q


def _plan(name, Q, P, k, kp, reorder, sms):
  """(S, query chunk, lists, tree merge?, merge region) of the kernel's plan, from the mirrors."""
  N, d, L, _, dpb, _ = CORPORA[name]
  S = tao.slices(Q, P, N, L, sms)
  qc = tao.query_chunk(Q, P, S, _layout(d, dpb)[0], k, kp, reorder)
  return S, qc, P * S, tao.tree_merge(P * S, kp, kp), tao.merge_region(P * S, kp, kp)


@pytest.mark.parametrize("name,Q,P,k,kp,reorder", SEARCH_CASES)
def test_search_at_every_slice_route_and_cap(corpus, name, Q, P, k, kp, reorder):
  ix = corpus(name)
  ix.check_build()
  es, _ = ix.search(_queries(name, Q, ix.x.shape[1]), P, k, kp, reorder)
  # where fewer rows are probed than k, the tail is (NaN, 0) on both paths
  probed = [int(np.diff(ix.ref["leaf_offsets"])[l].sum()) for l in
            tao.orc.topk_scan(_queries(name, Q, ix.x.shape[1]), ix.ref["centroids"], P)[1]]
  for r, n in enumerate(probed):
    assert np.isnan(es[r, min(n, k):]).all() and not np.isnan(es[r, :min(n, k)]).any()


def test_the_plan_mirror_matches_the_search_workspace():
  """The search workspace is a sum of the plan's buffers, so it pins S and the query chunk the kernel chose."""
  from recommenders_b200.ops import lib
  sms = _sms()
  a = lambda n: -(-n // 256) * 256
  for name, Q, P, k, kp, reorder in SEARCH_CASES + [("many_leaves", 4096, 10, 10, 2048, True)]:
    N, d, L, _, dpb, _ = CORPORA[name]
    S, qc, _, _, _ = _plan(name, Q, P, k, kp, reorder, sms)
    W = _layout(d, dpb)[1]
    parts = [qc * P * S * kp * 4, qc * P * S * kp * 8, qc * kp * 4, qc * kp * 8, qc * W * 128, qc * 4, qc * P * 4,
             qc * P * 8] + ([qc * k * 4, qc * k * 8] if reorder else [])
    want = sum(a(n) for n in parts) + lib().tfrs_topk_scan_workspace_bytes(qc, L, d, P)
    assert lib().tfrs_tree_ah_search_workspace_bytes(Q, d, L, P, dpb, k, kp, int(reorder), N) == want, name


def test_the_grid_reaches_every_edge():
  sms = _sms()
  plans = [(_plan(*c, sms), c) for c in SEARCH_CASES]
  S = {p[0] for p, _ in plans}
  assert {1, 2, 64} <= S and any(2 < s < 64 for s in S)
  assert any(p[2] == 64 and p[3] for p, _ in plans) and any(p[2] == 65 and not p[3] for p, _ in plans)
  limit = tao.MERGE_MAX_SMEM
  assert any(p[3] and limit - 1024 < p[4] * 24 <= limit for p, _ in plans)
  assert any(not p[3] and p[2] <= 64 and limit < p[4] * 24 <= limit + 1024 for p, _ in plans)
  assert any(c[2] == c[3] == c[4] == 2048 for _, c in plans)                        # k = k' = probes = 2048
  assert any(c[3] == 1 and c[4] == 2048 and c[5] for _, c in plans)                 # k = 1, k' = 2048
  assert any(c[2] > 64 and c[1] > p[1] and c[1] % p[1] for p, c in plans)           # uneven chunks, > 64 probes
  layouts = {(dpb,) + _layout(d, dpb) for d, dpb in WIDTHS}
  assert {(dpb, w) for dpb, _, _, w in layouts} == {(dpb, w) for dpb in range(1, 9) for w in range(1, dpb + 1)}
  Ws = {W for _, _, W, _ in layouts}
  assert {1, 32} <= Ws and len({W for W in Ws if W > 4}) >= 5
  # ta_lut's T[256 * 16] filled and ta_encode's largest shared memory, B * 16 * (dpb + 1) * 4 = 32 KB
  assert max(_layout(d, dpb)[0] * 16 for d, dpb in WIDTHS) == 256 * 16
  assert max(_layout(d, dpb)[0] * 16 * (dpb + 1) * 4 for d, dpb in WIDTHS) == 32 * 1024
  # the AH rowselect at W = 32 and k' = 2048: rowselect_cap(2048) * 12 + 32 * 128 = 53,248 B
  assert any(_layout(CORPORA[c[0]][1], CORPORA[c[0]][4])[1] == 32 and c[4] == 2048 for _, c in plans)


def test_no_queries():
  from recommenders_b200.layers import factorized_top_k as ftk
  x = _normal(500, 12, 3)
  for reorder in (None, 40):
    layer = ftk.TreeAH(k=10, num_leaves=5, num_leaves_to_search=2, num_reordering_candidates=reorder).index(cu(x))
    s, i = layer(cu(np.zeros((0, 12), F32)))
    assert tuple(s.shape) == (0, 10) and tuple(i.shape) == (0, 10)


def test_duplicate_centroids_leave_empty_leaves_that_are_probed(corpus):
  ix = corpus("repeated")
  sizes = np.diff(ix.ref["leaf_offsets"])
  assert (sizes == 0).sum() >= 50 and (sizes > 0).sum() <= 5
  probed = tao.orc.topk_scan(_queries("repeated", 3, 8), ix.ref["centroids"], 10)[1]
  assert all((sizes[p] == 0).any() for p in probed)
  assert len(np.unique(ix.ref["centroids"], axis=0)) <= 5


# ---- 5. the build kernels on adversarial inputs ------------------------------------------------------------------------
def _ints(shape, seed, lo=-2, hi=3):
  """Small integers as float32: every dot and squared norm is exact, so distinct centers tie exactly."""
  return np.random.default_rng(seed).integers(lo, hi, size=shape).astype(F32)


@pytest.mark.parametrize("n", [1, 65535, 65536, 65537, 131073])
def test_assign_breaks_ties_to_the_lower_center_across_chunks(n):
  from recommenders_b200 import ops
  c = _ints((7, 3), 1)
  centers = np.concatenate([c, c[::-1], c[:2]])     # every center twice or more
  x = _ints((n, 3), n)
  got = _np(ops.tree_ah_assign(cu(x), cu(centers)))
  np.testing.assert_array_equal(got, tao._aug_argmax(x, centers))


@pytest.mark.parametrize("pattern,n,L", [("first", 1, 1), ("first", 70000, 9), ("last", 70000, 9), ("last", 1000, 300),
                                         ("sparse", 70000, 5000), ("dense", 131073, 3)])
def test_group_offsets_and_order(pattern, n, L):
  from recommenders_b200 import ops
  rng = np.random.default_rng(n + L)
  leaf = {"first": np.zeros(n, np.int64), "last": np.full(n, L - 1, np.int64),
          "sparse": rng.choice(np.arange(0, L, 7), n), "dense": rng.integers(0, L, n)}[pattern]
  order, offsets = ops.tree_ah_group(cu(leaf), L)
  np.testing.assert_array_equal(_np(order), np.argsort(leaf, kind="stable"))
  np.testing.assert_array_equal(_np(offsets), np.concatenate([[0], np.cumsum(np.bincount(leaf, minlength=L))]))


def test_update_centroids_keeps_signed_zero_order_and_empty_leaves():
  from recommenders_b200 import ops
  from recommenders_b200.ops import lib, ptr, stream
  L, d = 6, 5
  x = _normal(3000, d, 5)
  leaf = np.random.default_rng(6).choice([1, 3, 5], 3000)
  zero = np.arange(0, 3000, 97)
  leaf[zero], x[zero] = 0, -0.0                     # leaf 0: only -0.0 members
  x[leaf == 3, 2] = np.tile(F32([1e8, 1.0, -1e8, 0.5]), 3000)[:(leaf == 3).sum()]   # order-sensitive sums
  cent = np.full((L, d), 7.25, F32)                 # leaves 2 and 4 are empty and keep this
  order, offsets = ops.tree_ah_group(cu(leaf.astype(np.int64)), L)
  got = cu(cent)
  tx = cu(x)
  ops.check(lib().tfrs_tree_ah_update_centroids_f32(ptr(tx), d, ptr(order), ptr(offsets), L, ptr(got), stream()), "")
  exp = tao.update_centroids(x, leaf, cent)
  assert _np(got).tobytes() == exp.tobytes()
  assert np.signbit(exp[0]).all() and np.all(exp[[2, 4]] == 7.25)


@pytest.mark.parametrize("n_train,d,dpb", [(1, 7, 3), (5, 7, 3), (16, 13, 8), (20, 256, 1), (40, 255, 8)])
def test_init_codebooks_repeats_rows_and_zeroes_unused_dims(n_train, d, dpb):
  """Fewer than 16 training rows: the 16 seed positions repeat (perm[arange(16) % n_train]), so centers start out equal.
  The last block's unused dims are written 0 over whatever the buffer held."""
  from recommenders_b200 import ops
  from recommenders_b200.ops import lib, ptr, stream
  L = 3
  x, cent = _normal(n_train, d, n_train), _normal(L, d, d)
  leaf = np.random.default_rng(7).integers(0, L, n_train)
  pos = np.random.default_rng(8).permutation(n_train)[np.arange(16) % n_train]
  B = _layout(d, dpb)[0]
  got = cu(np.full((B, 16, dpb), np.nan, F32))
  tx, tc, tp, tl = cu(x), cu(cent), cu(pos.astype(np.int64)), cu(leaf.astype(np.int64))
  ops.check(lib().tfrs_tree_ah_init_codebooks_f32(ptr(tx), d, ptr(tp), ptr(tl), ptr(tc), dpb, ptr(got), stream()), "")
  exp = np.zeros((B, 16, dpb), F32)
  r = (x - cent[leaf])[pos]
  for b, (c0, w) in enumerate(tao._blocks(d, dpb)):
    exp[b, :, :w] = r[:, c0:c0 + w]
  assert _np(got).tobytes() == exp.tobytes()


def _tied_codebooks(d, dpb, seed):
  """Integer centers with ties in every block: block 0 has 16 equal centers, every other block pairs j with 15 - j."""
  B = _layout(d, dpb)[0]
  cb = _ints((B, 16, dpb), seed)
  cb[0] = cb[0, 0]
  cb[1:, 8:] = cb[1:, 7::-1]
  return cb


@pytest.mark.parametrize("d,dpb,rows", [(7, 3, False), (7, 3, True), (100, 1, True), (256, 1, False), (255, 8, True),
                                        (61, 6, False)])
def test_encode_breaks_ties_to_the_lower_center_and_ignores_unused_dims(d, dpb, rows):
  """Exactly tied centers at every block and word (W up to 32, 32 KB of shared codebook at d = 256, dpb = 1); the last
  block's unused dims hold NaN, which must not reach any score."""
  from recommenders_b200 import ops
  n, L = 3000, 4
  x = _ints((n, d), d)
  cent = _ints((L, d), d + 1, -1, 2)
  leaf = np.random.default_rng(d).integers(0, L, n)
  perm = np.random.default_rng(d + 1).permutation(n).astype(np.int32) if rows else np.arange(n, dtype=np.int32)
  cb = _tied_codebooks(d, dpb, d + dpb)
  w_last = _layout(d, dpb)[2]
  cb[-1, :, w_last:] = np.nan
  got = ops.tree_ah_encode(cu(x), cu(perm) if rows else None, cu(leaf.astype(np.int64)), cu(cent), cu(cb), dpb)
  r = (x - cent[leaf])[perm]
  exp = tao.pack(tao._encode(r, cb, dpb))
  assert _np(got).tobytes() == exp.tobytes()
  codes = tao.unpack(exp, cb.shape[0])
  assert np.all(codes[:, 0] == 0) and np.all(codes[:, 1:] < 8)


@pytest.mark.parametrize("d,dpb", [(7, 3), (256, 1), (255, 8), (20, 6)])
def test_update_codebooks_keeps_centers_without_members(d, dpb):
  """Codes that leave centers 3 and 12 of every block (and all but center 0 of block 0) without members, residual
  blocks of -0.0, and the last block's unused dims, which must stay 0."""
  from recommenders_b200 import ops
  from recommenders_b200.ops import lib, ptr, stream
  n, L = 2000, 3
  B, _, w_last = _layout(d, dpb)
  x, cent = _normal(n, d, d), _normal(L, d, d + 1)
  leaf = np.random.default_rng(d).integers(0, L, n)
  codes = np.random.default_rng(d + 2).choice([j for j in range(16) if j not in (3, 12)], (n, B))
  codes[:, 0] = 0
  zero = codes[:, -1] == 5
  x[zero, (B - 1) * dpb:], cent[:, (B - 1) * dpb:] = -0.0, 0.0   # every residual of the last block coded 5 is -0.0
  cb = _normal(B * 16 * dpb, 1, 9).reshape(B, 16, dpb)
  cb[-1, :, w_last:] = 0
  got = cu(cb)
  tx, tl, tc, tw = cu(x), cu(leaf.astype(np.int64)), cu(cent), cu(tao.pack(codes))
  ops.check(lib().tfrs_tree_ah_update_codebooks_f32(ptr(tx), d, n, ptr(tl), ptr(tc), ptr(tw), dpb, ptr(got), stream()), "")
  exp = tao.update_codebooks(x - cent[leaf], codes, cb, dpb)
  assert _np(got).tobytes() == exp.tobytes()
  assert np.all(exp[:, [3, 12]] == cb[:, [3, 12]]) and np.signbit(exp[-1, 5, :w_last]).all()
  assert not np.any(exp[-1, :, w_last:])


# ---- 6. whole-layer builds at the size edges ---------------------------------------------------------------------------
@pytest.mark.parametrize("N,d,dpb,L,iters", [(1, 5, 3, 1, 0), (2, 5, 3, 2, 0), (15, 5, 3, 15, 0), (16, 5, 3, 16, 0),
                                             (17, 5, 3, 17, 0), (100000, 4, 2, 50, 2), (100001, 4, 2, 50, 2)])
def test_layer_builds_at_the_size_edges(N, d, dpb, L, iters):
  """N = L under 16 rows (repeated codebook seeds, so the first encode is all ties), no Lloyd steps, and the
  100,000-row training subset edge; then a search of every leaf, which pads when N < k."""
  from recommenders_b200.layers import factorized_top_k as ftk
  x = _normal(N, d, N)
  q = _normal(3, d, N + 1)
  P = min(L, 10)
  for reorder in (None, 20):
    layer = ftk.TreeAH(k=10, num_leaves=L, num_leaves_to_search=P, training_iterations=iters,
                       dimensions_per_block=dpb, num_reordering_candidates=reorder).index(cu(x))
    if reorder is None:
      exp = tao.build(x, L, iters, dpb)
      for key in INDEX_KEYS:
        assert _np(layer._index[key]).tobytes() == np.ascontiguousarray(exp[key]).tobytes(), key
    s, i = layer(cu(q))
    _same(s, i, *tao.search(exp, x, q, 10, P, dpb, reorder))
