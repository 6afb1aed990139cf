"""The per-bag float32 restatement of K11 in tests/test_gpu_embedding_bag_edges.py, checked on the CPU on the same edge
inputs its GPU cases use, so the bit-exact reference is not trusted blindly:
  - it agrees bit for bit (NaN by NaN-ness) with tests/embedding_bag_oracle.py, written separately, forward and backward;
  - a pooled sum stays within the recursive-summation bound gamma_n * sum |w*e| of a float64 evaluation of the same
    rule (plus one smallest subnormal per term for gradual underflow), and so does each D before its square root;
  - a mean / sqrtn output is the sum output divided by D in one float32 division, and a bag without a valid value is 0.
"""
import numpy as np
import pytest

import embedding_bag_oracle as ebo
import test_gpu_embedding_bag_edges as edges

f32 = np.float32
U = 2.0 ** -24                      # float32 unit roundoff


def _gamma(n):
  return n * U / (1 - n * U)


def _oracle(f):
  with np.errstate(all="ignore"):
    out, den = ebo.lookup(f.table, f.ids, f.splits, f.weights, f.combiner, f.L)
  return out.reshape(-1, f.table.shape[1]), den


CASES = dict(edges.ALL_CASES)


@pytest.mark.parametrize("case", sorted(CASES))
def test_restatement_agrees_with_the_oracle(case):
  rng = np.random.default_rng(1)
  for k, f in enumerate(CASES[case]()):
    out, den = edges.ref_forward(f)
    o_out, o_den = _oracle(f)
    edges.same(out, o_out, f"{case}: forward of feature {k}")
    if f.splits is not None and f.L == 0 and f.combiner != "sum":
      edges.same(den, o_den, f"{case}: D of feature {k}")
    g = rng.standard_normal(out.shape).astype(f32)
    with np.errstate(all="ignore"):
      exp = ebo.lookup_bwd(f.table.shape, f.ids, g, f.splits, f.weights, f.combiner, f.L)
    edges.same(edges.ref_backward(f, g), exp, f"{case}: backward of feature {k}")


def _float64_bags(f):
  """(sum w*e, sum |w*e|, the D sum, sum |D terms|, terms per bag) per pooled bag in float64: each product of two float32
  numbers is exact there."""
  table, ids, w, valid = edges._host(f)
  s0, s1 = edges.bag_bounds(f.splits, ids.size)
  dim = table.shape[1]
  B = s0.size
  acc, mag = np.zeros((B, dim)), np.zeros((B, dim))
  den, dmag, terms = np.zeros(B), np.zeros(B), np.zeros(B, np.int64)
  w64 = w.astype(np.float64)
  dterm = w64 if f.combiner == "mean" else w64 * w64
  for b in range(B):
    v = np.arange(s0[b], s1[b])[valid[s0[b]:s1[b]]]
    p = table[ids[v]].astype(np.float64) * w64[v, None]
    acc[b], mag[b] = p.sum(0), np.abs(p).sum(0)
    den[b], dmag[b] = dterm[v].sum(), np.abs(dterm[v]).sum()
    terms[b] = v.size
  return acc, mag, den, dmag, terms


@pytest.mark.parametrize("case", sorted(CASES))
def test_restatement_within_the_summation_bound(case):
  for k, f in enumerate(CASES[case]()):
    if f.splits is None or f.L > 0:
      continue
    acc64, mag, den64, dmag, terms = _float64_bags(f)
    acc32, _ = edges.ref_forward(f._replace(combiner="sum"))
    # float32 results of finite bags only; a subnormal product adds at most half the smallest subnormal per rounding
    ok = np.isfinite(acc32) & np.isfinite(mag) & (mag < 1e38)
    bound = (_gamma(terms)[:, None] * mag + terms[:, None] * 2.0 ** -149) * (1 + 1e-9)
    assert (np.abs(acc32.astype(np.float64) - acc64)[ok] <= bound[ok]).all(), (case, k)
    if f.combiner == "sum":
      continue
    out, den = edges.ref_forward(f)
    if f.combiner == "mean":
      dsum = den
    else:                  # sqrtn: the sum of w*w is the mean's D for weights w*w, and D is its rounded square root
      w = np.ones(f.ids.size, f32) if f.weights is None else f.weights.astype(f32)
      with np.errstate(over="ignore", under="ignore"):
        w2 = w * w
      _, dsum = edges.ref_forward(f._replace(combiner="mean", weights=w2))
      edges.same(den, np.sqrt(dsum), f"{case}: sqrtn D of feature {k}")
    dok = np.isfinite(dsum) & (dmag < 1e38)
    dbound = (_gamma(terms) * dmag + terms * 2.0 ** -149) * (1 + 1e-9)
    assert (np.abs(dsum.astype(np.float64) - den64)[dok] <= dbound[dok]).all(), (case, k)
    # one division of the sum by D; nothing divided in a bag without a valid value
    with np.errstate(divide="ignore", invalid="ignore", over="ignore", under="ignore"):
      q = np.where((terms > 0)[:, None], acc32 / den[:, None], acc32).astype(f32)
    edges.same(out, q, f"{case}: feature {k} as sum / D")
    assert (out[terms == 0] == 0).all() and not np.signbit(out[terms == 0]).any()


def test_edge_inputs_reach_their_edges():
  """The shared inputs hold what the GPU cases claim: every bag length 0..13, empty runs, splits after 0 and before n,
  32-bit aliases of valid rows, subnormal weights and -0.0 entries."""
  rng = np.random.default_rng(0)
  lens = edges.every_length(rng)
  assert set(range(14)) <= set(lens.tolist()) and lens[0] == lens[1] == 0 and lens[-1] == 0
  walk = edges.batch_walk_case("mean")[0]
  s0, s1 = edges.bag_bounds(walk.splits, walk.ids.size)
  valid = (walk.ids >= 0) & (walk.ids < walk.table.shape[0])
  counts = np.array([valid[a:z].sum() for a, z in zip(s0, s1)])
  assert ((counts == 0) & (s1 > s0)).sum() >= 10
  for pos in range(edges.BG_BATCH):
    assert any(z - a > pos and not valid[a + pos] and valid[a:z].sum() == z - a - 1 for a, z in zip(s0, s1)), pos
  for n_bags in (1, 16, 1025):
    f = edges.splits_case(n_bags, n_bags)[0]
    s0, s1 = edges.bag_bounds(f.splits, f.ids.size)
    assert s0[0] > 0 and s1[-1] < f.ids.size and len(s0) == n_bags
  ids = edges.id_case(np.int64)[0].ids
  rows = edges.id_case(np.int64)[0].table.shape[0]
  alias = ids.astype(np.int32).astype(np.int64)
  assert ((ids >= rows) & (alias >= 0) & (alias < rows)).sum() >= 3
  w = edges.weight_case("zero, negative and subnormal weights")[0].weights
  assert ((w != 0) & (np.abs(w) < np.finfo(f32).tiny)).sum() >= 3
  t = edges.weight_case("signed zeros")[0].table
  assert np.signbit(t[t == 0]).sum() > 0
