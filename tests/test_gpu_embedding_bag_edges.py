"""K11 (TPUEmbedding's bag kernels, csrc/embedding_bag.cu) at its edges, bit for bit against a plain reference.

The reference is restated here, per bag, in float32 (DESIGN.md section 2, A16), independently of
tests/embedding_bag_oracle.py:
  - pooled: acc = acc + w*e over the bag's valid values in value order from +0.0f, one rounding per multiply and one per
    add; D = 1 (sum), sum w (mean) or sqrtf(sum w*w) (sqrtn), summed the same way; out = acc / D as one division (none
    for sum, none for a bag without a valid value, which gives zeros);
  - sequence: position j of bag b is w_j * e_j for j < min(L, bag size), zeros elsewhere;
  - dense: row i is e_i;
  - backward: (g_b * w) / D_b for a pooled value (g_b * w for sum), g_{b,j} * w for a sequence value (zeros past L), g_i
    for a dense value;
  - ids outside [0, rows) are dropped with their weights: nothing added to the bag or to D, a zero row.
Every output, denominator and gradient row is compared by its bits; NaN only by NaN-ness (the GPU's canonical NaN is
0x7fffffff, x86's 0xffc00000).  tests/test_embedding_bag_oracle_edges.py checks this restatement itself on the CPU.

The cases reach what the random shapes of tests/test_gpu_tpu_embedding.py do not: every row width class of both the
float4 and the scalar path, the scalar path forced at aligned widths, every bag length residue of the 4-value batch,
empty-bag runs around the backward's binary search, row splits that start after 0 or end before n, int64 ids that
would alias a row if truncated to 32 bits, signed zeros, zero and subnormal weights, zero denominators, sequence
cuts, the 128-feature launch groups with exact launch counts, strided outputs and gradients, and each argument error.
"""
from typing import NamedTuple, Optional

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

f32 = np.float32
INT64_MIN, INT64_MAX = -2**63, 2**63 - 1
INT32_MIN, INT32_MAX = -2**31, 2**31 - 1
BG_MAX_FEATURES = 128     # features per launch in csrc/embedding_bag.cu
BG_BATCH = 4              # pooled values per batch of row loads
NAN_FILL = np.uint32(0x7FC00123)        # a quiet NaN with a payload: what the kernels do not write keeps these bits
ID_FILL = -0x5A5A5A5A5A5A5A5B


# ---- the reference -----------------------------------------------------------------------------------------------------
class Feat(NamedTuple):
  """One feature in host arrays: ids (int32 / int64), row splits (None: dense), weights (None: all 1), combiner and
  max sequence length L (> 0: a sequence feature)."""
  table: np.ndarray
  ids: np.ndarray
  splits: Optional[np.ndarray] = None
  weights: Optional[np.ndarray] = None
  combiner: str = "mean"
  L: int = 0


def out_rows(f: Feat) -> int:
  if f.splits is None:
    return f.ids.size
  return (len(f.splits) - 1) * (f.L if f.L > 0 else 1)


def bag_bounds(splits, n):
  """Bag b holds values [s0, s1): its splits clamped to [0, n], and s1 >= s0."""
  sp = np.asarray(splits, np.int64)
  s0 = np.minimum(np.maximum(sp[:-1], 0), n)
  s1 = np.minimum(np.maximum(sp[1:], s0), n)
  return s0, s1


def _host(f: Feat):
  table = np.asarray(f.table, f32)
  ids = np.asarray(f.ids).astype(np.int64).reshape(-1)
  w = np.ones(ids.size, f32) if f.weights is None else np.asarray(f.weights, f32).reshape(-1)
  valid = (ids >= 0) & (ids < table.shape[0])
  return table, ids, w, valid


def ref_forward(f: Feat):
  """(output rows [out_rows, dim], per-bag D for pooled mean / sqrtn, else None)."""
  table, ids, w, valid = _host(f)
  n, dim = ids.size, table.shape[1]
  e = np.zeros((n, dim), f32)
  e[valid] = table[ids[valid]]
  if f.splits is None:
    return e, None
  s0, s1 = bag_bounds(f.splits, n)
  B, lens = s0.size, s1 - s0
  if f.L > 0:
    out = np.zeros((B * f.L, dim), f32)
    for j in range(f.L):                                      # position j of every bag that has one
      b = np.nonzero(lens > j)[0]
      v = s0[b] + j
      b, v = b[valid[v]], v[valid[v]]
      with np.errstate(over="ignore", under="ignore", invalid="ignore"):
        out[b * f.L + j] = e[v] * w[v, None]
    return out, None
  with np.errstate(over="ignore", under="ignore", invalid="ignore"):
    prod = e * w[:, None]                                     # one rounding per multiply
    dw = w if f.combiner == "mean" else w * w
  acc = np.zeros((B, dim), f32)
  den = np.zeros(B, f32)
  short = lens <= 64
  with np.errstate(over="ignore", invalid="ignore"):
    for j in range(int(lens[short].max(initial=0))):         # short bags: the j-th value of each, in value order
      b = np.nonzero(short & (lens > j))[0]
      v = s0[b] + j
      b, v = b[valid[v]], v[valid[v]]                         # a dropped id adds nothing
      acc[b] = acc[b] + prod[v]
      den[b] = den[b] + dw[v]
    for b in np.nonzero(~short)[0]:                           # long bags: a running sum from a leading +0.0 row
      v = np.arange(s0[b], s1[b])[valid[s0[b]:s1[b]]]
      acc[b] = np.add.accumulate(np.vstack([np.zeros((1, dim), f32), prod[v]]), axis=0, dtype=f32)[-1]
      den[b] = np.add.accumulate(np.concatenate([np.zeros(1, f32), dw[v]]), dtype=f32)[-1]
  if f.combiner == "sum":
    return acc, None
  if f.combiner == "sqrtn":
    den = np.sqrt(den)
  counts = np.concatenate([[0], np.cumsum(valid)])
  some = counts[s1] - counts[s0] > 0                          # a bag without a valid value is not divided
  out = acc.copy()
  with np.errstate(divide="ignore", invalid="ignore", over="ignore", under="ignore"):
    out[some] = acc[some] / den[some, None]                   # one division
  return out, den


def ref_backward(f: Feat, grad):
  """The gradient rows [n, dim] of the feature's values from the gradient of its output rows [out_rows, dim]."""
  table, ids, w, valid = _host(f)
  n, dim = ids.size, table.shape[1]
  g = np.asarray(grad, f32).reshape(-1, dim)
  out = np.zeros((n, dim), f32)
  if f.splits is None:
    out[valid] = g[valid]
    return out
  s0, s1 = bag_bounds(f.splits, n)
  lens = s1 - s0
  bag = np.full(n, -1, np.int64)                              # the bag holding each value, -1 for none
  first = np.repeat(s0, lens)
  bag[first + (np.arange(lens.sum()) - np.repeat(np.cumsum(lens) - lens, lens))] = np.repeat(np.arange(s0.size), lens)
  m = valid & (bag >= 0)
  v, b = np.nonzero(m)[0], bag[m]
  with np.errstate(divide="ignore", invalid="ignore", over="ignore", under="ignore"):
    if f.L > 0:
      j = v - s0[b]
      v, b, j = v[j < f.L], b[j < f.L], j[j < f.L]            # values past L keep zero rows
      out[v] = g[b * f.L + j] * w[v, None]
    elif f.combiner == "sum":
      out[v] = g[b] * w[v, None]
    else:
      _, den = ref_forward(f._replace(table=table[:, :1]))
      out[v] = (g[b] * w[v, None]) / den[b, None]
  return out


# ---- case inputs (shared with tests/test_embedding_bag_oracle_edges.py) ------------------------------------------------
def splits_of(lens, start=0):
  return (start + np.concatenate([[0], np.cumsum(lens)])).astype(np.int64)


def dropped_pool(rows, dtype):
  """Ids a feature of `rows` rows must drop; the int64 ones alias a valid row when truncated to 32 bits."""
  if np.dtype(dtype) == np.int32:
    return np.array([-1, rows, rows + 1, INT32_MIN, INT32_MAX], np.int64)
  return np.array([-1, rows, rows + 1, INT64_MIN, INT64_MAX, 2**31, 2**32 + 3, 2**32, 2**33 + 1], np.int64)


def rand_ids(rng, n, rows, dtype=np.int64, p_drop=0.15):
  ids = rng.integers(0, rows, size=n).astype(np.int64)
  k = rng.random(n) < p_drop
  ids[k] = rng.choice(dropped_pool(rows, dtype), size=int(k.sum()))
  return ids.astype(dtype)


def every_length(rng, extra=20, top=13):
  """Every bag length 0..top, then random ones; empty runs at the start, in the middle and at the end."""
  lens = [0, 0] + list(range(top + 1)) + [0, 0, 0, 5] + list(rng.integers(0, top + 1, size=extra)) + [0, 1, 0, 0]
  return np.array(lens, np.int64)


def width_case(dim, combiner, seed):
  """Pooled (int32, weighted), pooled (int64), sequence (L = 5, weighted) and dense (int64 [n, 3]) on two tables."""
  rng = np.random.default_rng(seed)
  t1 = rng.standard_normal((37, dim)).astype(f32)
  t2 = rng.standard_normal((11, dim)).astype(f32)
  lens = every_length(rng)
  sp, n = splits_of(lens), int(lens.sum())
  lens2 = every_length(rng)
  sp2, n2 = splits_of(lens2), int(lens2.sum())
  return [Feat(t1, rand_ids(rng, n, 37, np.int32), sp, rng.uniform(-1, 2, size=n).astype(f32), combiner),
          Feat(t2, rand_ids(rng, n2, 11), sp2, None, combiner),
          Feat(t1, rand_ids(rng, n, 37), sp, rng.uniform(-1, 2, size=n).astype(f32), combiner, 5),
          Feat(t2, rand_ids(rng, 3 * 13 + seed % 4, 11).reshape(-1), None)]


def batch_walk_case(combiner, seed=5):
  """Bags of every length 0..13 with dropped ids at each position of a 4-value batch, a whole batch dropped, and bags
  of only dropped ids."""
  rng = np.random.default_rng(seed)
  rows, dim = 29, 12
  table = rng.standard_normal((rows, dim)).astype(f32)
  bags = []
  for length in range(14):
    bags.append(rng.integers(0, rows, size=length))
    for pos in range(min(length, 2 * BG_BATCH)):          # one dropped id at each position of the first two batches
      b = rng.integers(0, rows, size=length)
      b[pos] = -1 if pos % 2 else rows + pos
      bags.append(b)
  for length in (4, 8, 9, 13):
    b = rng.integers(0, rows, size=length)
    b[:4] = [-1, rows, INT64_MIN, 2**32 + 3]              # the first batch wholly dropped
    bags.append(b)
    c = rng.integers(0, rows, size=length)
    c[4:8] = -7                                           # the second batch wholly dropped
    bags.append(c)
  for length in (1, 3, 4, 5, 12):
    bags.append(np.full(length, rows))                    # nothing valid: zeros, D = 0
    bags.append(rng.choice(dropped_pool(rows, np.int64), size=length))
  lens = np.array([len(b) for b in bags], np.int64)
  ids = np.concatenate(bags).astype(np.int64)
  w = rng.uniform(0.25, 2, size=ids.size).astype(f32)
  return [Feat(table, ids, splits_of(lens), w, combiner), Feat(table, ids.copy(), splits_of(lens), None, combiner)]


def middle_run(n_bags):
  return n_bags // 2 - 1


def splits_case(n_bags, seed):
  """n_bags bags with runs of empty bags at the start, in the middle, at the end and directly before non-empty bags; a
  first split after 0 and a last split before n, so values outside every bag remain."""
  rng = np.random.default_rng(seed)
  rows, dim = 50, 8
  table = rng.standard_normal((rows, dim)).astype(f32)
  lens = rng.integers(0, 6, size=n_bags)
  lens[0] = max(lens[0], 1)
  if n_bags >= 8:                                    # empty runs at both ends, each beside a non-empty bag
    lens[:3], lens[-2:] = 0, 0
    lens[3], lens[-3] = max(lens[3], 1), max(lens[-3], 1)
  if n_bags >= 12:                                   # and one in the middle, directly before a non-empty bag
    m = middle_run(n_bags)
    lens[m:m + 3], lens[m + 3] = 0, 4
  head, tail = 3, 2
  sp = splits_of(lens, start=head)
  n = int(sp[-1]) + tail
  ids = rand_ids(rng, n, rows)
  w = rng.uniform(-1, 2, size=n).astype(f32)
  return [Feat(table, ids, sp, w, c) for c in ("sum", "mean", "sqrtn")] + [Feat(table, ids, sp, w, "mean", 3)]


def id_case(dtype):
  """Ids at -1, rows - 1, rows and the 32-bit aliases of valid rows, pooled, sequence and dense."""
  rows, dim = 7, 8
  table = np.arange(rows * dim, dtype=f32).reshape(rows, dim) / 8 + 1
  edge = [-1, 0, rows - 1, rows, 3, rows + 1]
  if np.dtype(dtype) == np.int64:
    edge += [2**31, 2**32 + 3, 2**32, INT64_MIN, INT64_MAX, 2**31 - 1, 2**32 + rows - 1, -2**32 + 3]
  else:
    edge += [INT32_MIN, INT32_MAX, INT32_MAX - 1, INT32_MIN + 3]
  ids = np.array(edge, np.int64).astype(dtype)
  lens = [1] * len(edge) + [len(edge)]
  ids = np.concatenate([ids, ids])
  sp = splits_of(lens)
  w = np.linspace(0.5, 2, ids.size).astype(f32)
  return [Feat(table, ids, sp, w, "mean"), Feat(table, ids, sp, w, "sqrtn"), Feat(table, ids, sp, None, "sum"),
          Feat(table, ids, sp, w, "mean", 4), Feat(table, ids, None)]


def weight_case(which):
  """Weights and values at the edges of the arithmetic."""
  rows, dim = 6, 8
  rng = np.random.default_rng(len(which))
  table = rng.standard_normal((rows, dim)).astype(f32)
  if which == "zero, negative and subnormal weights":
    ids = np.array([0, 1, 2, 3, 4, 5, 0, 1, 2, 3, 1, 2], np.int64)
    w = np.array([0, -1.5, 1e-40, -3e-39, 0, 2, 1e-45, -0.0, 0.5, -2, 1e-38, 7e-46], f32)
    lens = [2, 2, 3, 1, 2, 2]
  elif which == "mean with a zero weight sum":
    ids = np.array([0, 1, 2, 2, 3, 4, 5, 1], np.int64)
    w = np.array([1, -1, 0.5, -0.5, 0, 0, 2, -2], f32)
    lens = [2, 2, 2, 2]
  elif which == "sqrtn with w*w underflowing":
    ids = np.array([0, 1, 2, 3, 4, 5], np.int64)
    w = np.array([1e-23, -1e-23, 3e-30, 1e-20, 1e-40, 1.0], f32)
    lens = [2, 1, 1, 1, 1]
    table[2, :2] = 0
  elif which == "overflow":
    ids = np.array([0, 1, 2, 3, 4, 5, 0], np.int64)
    w = np.array([3e38, 3e38, 1e30, -3e38, 3.4e38, 3.4e38, 1], f32)
    table[:] = np.abs(table) + 1
    table[3] = -table[3]
    lens = [2, 2, 3]
  elif which == "signed zeros":
    table[:] = -0.0
    table[4] = [0.0, -0.0, 1, -1, -0.0, 0, 2, -2]
    ids = np.array([0, 1, 2, 4, 0, 5, 5, 3], np.int64)
    w = np.array([1, 1, -1, 1, 2, 1, -1, 0.5], f32)
    lens = [1, 2, 1, 2, 2]
  else:
    raise KeyError(which)
  sp = splits_of(lens)
  feats = [Feat(table, ids, sp, w, c) for c in ("sum", "mean", "sqrtn")]
  return feats + [Feat(table, ids, sp, w, "mean", 2), Feat(table, ids, sp, w, "sum", 3), Feat(table, ids, None)]


WEIGHT_CASES = ["zero, negative and subnormal weights", "mean with a zero weight sum", "sqrtn with w*w underflowing",
                "overflow", "signed zeros"]


def sequence_case(seed=7):
  """L = 1 and L below, equal to and above the bag lengths; dropped ids mid-bag; weights on every position."""
  rng = np.random.default_rng(seed)
  rows, dim = 13, 12
  table = rng.standard_normal((rows, dim)).astype(f32)
  lens = np.array([0, 1, 2, 3, 4, 5, 6, 0, 7, 9, 4], np.int64)
  ids = rng.integers(0, rows, size=int(lens.sum())).astype(np.int64)
  sp = splits_of(lens)
  ids[sp[4] + 1] = -1                 # mid-bag in a 4-value bag
  ids[sp[8] + 2] = rows               # and in a 7-value bag
  ids[sp[9] + 0] = 2**32 + 1
  w = rng.uniform(-2, 2, size=ids.size).astype(f32)
  return [Feat(table, ids, sp, w, "mean", L) for L in (1, 3, 4, 7, 12)]


ALL_CASES = ([(f"width {d} {c}", lambda d=d, c=c: width_case(d, c, d)) for d in (1, 3, 4, 7, 8, 33, 132)
              for c in ("sum", "mean", "sqrtn")] +
             [(f"batch walk {c}", lambda c=c: batch_walk_case(c)) for c in ("sum", "mean", "sqrtn")] +
             [(f"splits {b}", lambda b=b: splits_case(b, b)) for b in (1, 2, 3, 8, 15, 16, 17, 64, 65)] +
             [("ids int32", lambda: id_case(np.int32)), ("ids int64", lambda: id_case(np.int64))] +
             [(w, lambda w=w: weight_case(w)) for w in WEIGHT_CASES] +
             [("sequence", sequence_case)])


# ---- GPU helpers -------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def tfrs():
  import recommenders_b200 as t
  return t


def same(got, exp, what=""):
  """Bit equality; NaN compared by NaN-ness only."""
  got = got.detach().cpu().numpy() if isinstance(got, torch.Tensor) else np.asarray(got)
  exp = np.ascontiguousarray(exp)
  assert got.shape == exp.shape and got.dtype == exp.dtype, (what, got.shape, got.dtype, exp.shape, exp.dtype)
  if got.dtype.kind != "f":
    np.testing.assert_array_equal(got, exp, err_msg=what)
    return
  gn, en = np.isnan(got), np.isnan(exp)
  assert np.array_equal(gn, en), f"{what}: NaN at {np.argwhere(gn != en)[:5].tolist()}"
  bits = np.dtype(f"u{got.itemsize}")
  gb, eb = np.where(gn, 0, got.view(bits)), np.where(en, 0, exp.view(bits))
  if not np.array_equal(gb, eb):
    bad = np.argwhere(gb != eb)[:5].tolist()
    raise AssertionError(f"{what}: bits differ at {bad}: got {[got[tuple(i)] for i in bad]}, "
                         f"expected {[exp[tuple(i)] for i in bad]}")


def filled(shape, fill=NAN_FILL):
  return torch.from_numpy(np.full(shape, fill, np.uint32).view(f32)).cuda()


def dev(a):
  return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def expected_launches(feats):
  """(forward, backward) launches: per group of 128 whole features, one forward launch when any feature has output
  rows or values, one backward launch when any feature has values."""
  fwd = bwd = 0
  for k in range(0, len(feats), BG_MAX_FEATURES):
    grp = feats[k:k + BG_MAX_FEATURES]
    fwd += any(out_rows(f) > 0 or f.ids.size > 0 for f in grp)
    bwd += any(f.ids.size > 0 for f in grp)
  return fwd, bwd


def run_ops(tfrs, feats, outs=None, col_offs=None, tables=None, grads=None, grad_rows=None, seed=0, launches=None):
  """One ops.embedding_bag call and one ops.embedding_bag_bwd call, everything against the reference: the outputs at
  each feature's columns (other columns keep what they held), the ids, the denominators (left alone for sum), the
  gradient rows and the exact launch counts.  `outs[k]` (shared by features that pass the same tensor), `col_offs[k]`,
  `tables[k]`, `grads[k]` and `grad_rows[k]` replace the defaults: fresh NaN-filled [out_rows, dim] outputs at column
  0, uploaded tables, random contiguous gradients and NaN-filled gradient rows.  Returns (outputs, gradient rows)."""
  ops = tfrs.ops
  rng = np.random.default_rng(seed)
  K = len(feats)
  if tables is None:                                          # one upload per distinct host table
    up = {}
    tables = [up[id(f.table)] if id(f.table) in up else up.setdefault(id(f.table), dev(f.table)) for f in feats]
  col_offs = col_offs or [0] * K
  outs = outs or [filled((out_rows(f), f.table.shape[1])) for f in feats]
  before = {id(o): o.cpu().numpy().copy() for o in outs}
  exp_out = {id(o): before[id(o)].copy() for o in outs}
  bf, exp_den = [], []
  for f, t, o, c in zip(feats, tables, outs, col_offs):
    ids = torch.full((f.ids.size,), ID_FILL, dtype=torch.int64, device="cuda")
    den = filled((len(f.splits) - 1,)) if f.splits is not None and f.L == 0 else None
    bf.append(ops.BagFeature(t, dev(f.ids), o, None if f.splits is None else dev(f.splits),
                             None if f.weights is None else dev(f.weights), f.combiner, f.L, c, ids, den))
    r, d = ref_forward(f)
    exp_out[id(o)][:, c:c + f.table.shape[1]] = r
    exp_den.append(d)
  torch.cuda.synchronize()
  n0 = ops.launch_count()
  ops.embedding_bag(bf)
  n1 = ops.launch_count()
  for k, (f, b) in enumerate(zip(feats, bf)):
    same(b.out, exp_out[id(b.out)], f"output of feature {k}")
    same(b.ids, f.ids.astype(np.int64).reshape(-1), f"ids of feature {k}")
    if b.denom is not None:
      same(b.denom, exp_den[k] if exp_den[k] is not None else np.full(b.denom.shape, NAN_FILL, np.uint32).view(f32),
           f"denominators of feature {k}")
  grads = grads or [dev(rng.standard_normal((out_rows(f), f.table.shape[1])).astype(f32)) for f in feats]
  grad_rows = grad_rows or [filled((f.ids.size, f.table.shape[1])) for f in feats]
  n2 = ops.launch_count()
  ops.embedding_bag_bwd(bf, grads, grad_rows)
  n3 = ops.launch_count()
  for k, (f, g, gr, c) in enumerate(zip(feats, grads, grad_rows, col_offs)):
    same(gr, ref_backward(f, g.cpu().numpy()[:, c:c + f.table.shape[1]]), f"gradient rows of feature {k}")
  assert (n1 - n0, n3 - n2) == (launches or expected_launches(feats))
  return [b.out for b in bf], grad_rows


# ---- 1. row widths -----------------------------------------------------------------------------------------------------
VEC_DIMS = [4 * q for q in (1, 2, 3, 5, 7, 8, 25, 32, 33, 64, 256)]
SCALAR_DIMS = [1, 2, 3, 5, 7, 9, 33, 127, 1001]


@pytest.mark.parametrize("combiner", ["sum", "mean", "sqrtn"])
@pytest.mark.parametrize("dim", VEC_DIMS + SCALAR_DIMS)
def test_row_widths(tfrs, dim, combiner):
  """dim/4 of 1 .. 256 on the float4 path and odd widths on the scalar path: the e / P4 split of both kernels, rows wider
  than a CTA, and the backward's 4-item tail; pooled, sequence and dense features in one launch each way."""
  run_ops(tfrs, width_case(dim, combiner, dim), seed=dim)


# ---- 2. the scalar path at aligned widths ----------------------------------------------------------------------------------
SCALAR_REASONS = ["ld % 4", "col_off % 4", "table + 1 float", "out + 1 float", "grad + 1 float", "grad_rows + 1 float"]


@pytest.mark.parametrize("reason", SCALAR_REASONS)
@pytest.mark.parametrize("dim", [4, 8, 36, 128])
def test_forced_scalar_path(tfrs, dim, reason):
  """dim % 4 == 0 with one misaligned piece takes the scalar path; the bits are those of the float4 path."""
  feats = width_case(dim, "sqrtn", 1000 + dim)
  rng = np.random.default_rng(dim)
  grads_h = [rng.standard_normal((out_rows(f), dim)).astype(f32) for f in feats]
  vec_out, vec_rows = run_ops(tfrs, feats, grads=[dev(g) for g in grads_h])

  def shifted(shape, fill=None):
    flat = filled((int(np.prod(shape)) + 4,)) if fill is None else torch.zeros(int(np.prod(shape)) + 4, device="cuda")
    return flat[1:1 + int(np.prod(shape))].view(*shape)

  K = len(feats)
  outs = col_offs = tables = grads = grad_rows = None
  if reason == "ld % 4":
    outs = [filled((out_rows(f), dim + 1)) for f in feats]
  elif reason == "col_off % 4":
    outs, col_offs = [filled((out_rows(f), dim + 4)) for f in feats], [2] * K
  elif reason == "table + 1 float":
    tables = []
    for f in feats:
      t = shifted(f.table.shape, 0)
      t.copy_(dev(f.table))
      tables.append(t)
  elif reason == "out + 1 float":
    outs = [shifted((out_rows(f), dim)) for f in feats]
  elif reason == "grad + 1 float":
    grads = []
    for g in grads_h:
      t = shifted(g.shape, 0)
      t.copy_(dev(g))
      grads.append(t)
  else:
    grad_rows = [shifted((f.ids.size, dim)) for f in feats]
  if grads is None:
    c = col_offs or [0] * K
    grads = []
    for g, o, off in zip(grads_h, outs or [None] * K, c):
      full = np.zeros((g.shape[0], dim if o is None else o.shape[1]), f32)
      full[:, off:off + dim] = g
      grads.append(dev(full))
  got_out, got_rows = run_ops(tfrs, feats, outs=outs, col_offs=col_offs, tables=tables, grads=grads,
                              grad_rows=grad_rows)
  c = col_offs or [0] * K
  for k in range(K):
    same(got_out[k][:, c[k]:c[k] + dim], vec_out[k].cpu().numpy(), f"output {k}, scalar against float4 path")
    same(got_rows[k], vec_rows[k].cpu().numpy(), f"gradient rows {k}, scalar against float4 path")


# ---- 3. the bag walk ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("combiner", ["sum", "mean", "sqrtn"])
def test_bag_walk(tfrs, combiner):
  """Every bag length 0..13, a dropped id at each position of a batch, whole batches dropped, and bags with nothing
  valid (zeros, D = 0, zero gradient rows)."""
  run_ops(tfrs, batch_walk_case(combiner))


def test_long_bag_beside_short_ones(tfrs):
  """One 100 000-value bag beside 5000 one-value bags in one launch: one thread group walks 25 000 batches in order."""
  rng = np.random.default_rng(21)
  rows, dim = 1000, 16
  table = rng.standard_normal((rows, dim)).astype(f32)
  lens = np.ones(5001, np.int64)
  lens[2500] = 100_000
  n = int(lens.sum())
  ids = rand_ids(rng, n, rows, p_drop=0.01)
  w = rng.uniform(0, 1, size=n).astype(f32)
  feats = [Feat(table, ids, splits_of(lens), w, c) for c in ("sum", "mean", "sqrtn")]
  run_ops(tfrs, feats + [Feat(table, rand_ids(rng, 1, rows), np.array([0, 1], np.int64), None, "mean")])


# ---- 4. row splits -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n_bags", [1, 2, 3, 4, 5, 7, 8, 9, 15, 16, 17, 1023, 1024, 1025])
def test_row_splits(tfrs, n_bags):
  """n_bags at the binary search's power-of-two bounds; empty-bag runs at the start, in the middle (directly before a
  non-empty bag) and at the end; splits that start at 3 and end 2 values before n."""
  feats = splits_case(n_bags, n_bags)
  s0, s1 = bag_bounds(feats[0].splits, feats[0].ids.size)
  assert s0[0] > 0 and s1[-1] < feats[0].ids.size
  if n_bags >= 8:
    assert (s1 == s0)[:3].all() and (s1 == s0)[-2:].all() and s1[3] > s0[3] and s1[-3] > s0[-3]
  if n_bags >= 12:
    m = middle_run(n_bags)
    assert (s1 == s0)[m:m + 3].all() and s1[m + 3] > s0[m + 3] == s0[m]
  run_ops(tfrs, feats, seed=n_bags)


# ---- 5. ids --------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", ["int32", "int64"])
def test_ids(tfrs, dtype):
  """-1, rows - 1, rows and, for int64, 2^31, 2^32 + 3, -2^63 and 2^63 - 1 (row 3 or 0 if truncated to 32 bits) are
  dropped, and every one of them is copied to the ids of the backward pair."""
  run_ops(tfrs, id_case(np.dtype(dtype)))


# ---- 6. weights and values ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("which", WEIGHT_CASES)
def test_weights_and_values(tfrs, which):
  """Zero, negative and subnormal weights; mean with sum w = 0 and sqrtn with w*w underflowing to D = 0 (inf and NaN);
  overflow to inf; table entries of -0.0 (a pooled bag gives +0.0, sequence and dense positions keep -0.0)."""
  feats = weight_case(which)
  outs, _ = run_ops(tfrs, feats)
  if which == "signed zeros":
    pooled = outs[0].cpu().numpy()
    assert np.signbit(pooled[0]).sum() == 0                          # one -0.0 row pooled: +0.0
    assert np.signbit(outs[5].cpu().numpy()[0]).all()                 # dense keeps -0.0
    assert np.signbit(outs[3].cpu().numpy()[0]).all()                 # so does a sequence position with w = 1
  if which in ("mean with a zero weight sum", "sqrtn with w*w underflowing", "overflow"):
    assert not np.isfinite(np.concatenate([o.cpu().numpy().ravel() for o in outs[:3]])).all()


# ---- 7. sequence features ----------------------------------------------------------------------------------------------------
def test_sequence_cuts(tfrs):
  """L = 1 and L below, equal to and above the bag lengths; a dropped id leaves a zero at its position (later values do
  not move up); values past L get zero gradient rows; a weight on every position."""
  feats = sequence_case()
  outs, rows = run_ops(tfrs, feats)
  f = feats[2]                                                          # L = 4
  b = 4
  o = outs[2].cpu().numpy().reshape(-1, 4, f.table.shape[1])
  assert (o[b, 1] == 0).all() and (o[b, 2] != 0).any()                  # position 1 dropped, position 2 kept
  r = rows[0].cpu().numpy()                                             # L = 1: only each bag's first value has a row
  s0, s1 = bag_bounds(f.splits, f.ids.size)
  later = np.concatenate([np.arange(a + 1, z) for a, z in zip(s0, s1)])
  assert (r[later] == 0).all()


# ---- 8. launch groups ----------------------------------------------------------------------------------------------------
def _mixed_features(rng, count, tables):
  """`count` small features cycling through pooled, sequence and dense kinds over shared tables."""
  feats = []
  for k in range(count):
    t = tables[k % len(tables)]
    rows = t.shape[0]
    kind = k % 3
    if kind == 2:
      feats.append(Feat(t, rand_ids(rng, 1 + k % 5, rows, np.int32 if k % 2 else np.int64)))
      continue
    lens = rng.integers(0, 4, size=1 + k % 4)
    lens[0] = max(lens[0], 1)
    n = int(lens.sum())
    feats.append(Feat(t, rand_ids(rng, n, rows), splits_of(lens), rng.uniform(0, 2, size=n).astype(f32),
                      ("sum", "mean", "sqrtn")[k % 3], 2 if kind == 1 else 0))
  return feats


@pytest.mark.parametrize("count", [1, 127, 128, 129, 256, 257])
def test_launch_groups(tfrs, count):
  """Exactly one launch each way per group of 128 features, pooled, sequence and dense mixed."""
  rng = np.random.default_rng(count)
  tables = [rng.standard_normal((r, d)).astype(f32) for r, d in ((17, 4), (9, 3), (23, 8))]
  feats = _mixed_features(rng, count, tables)
  g = -(-count // BG_MAX_FEATURES)
  assert expected_launches(feats) == (g, g)
  run_ops(tfrs, feats, seed=count, launches=(g, g))


def test_very_different_sizes_in_one_launch(tfrs):
  """n = 1 beside n = 10^6 (dense), a 250 000-bag pooled feature and a sequence feature, in one launch each way."""
  rng = np.random.default_rng(22)
  table = rng.standard_normal((5000, 8)).astype(f32)
  big = rand_ids(rng, 10**6, 5000, p_drop=0.01)
  lens = rng.integers(0, 4, size=250_000)
  n = int(lens.sum())
  feats = [Feat(table, rand_ids(rng, 1, 5000)), Feat(table, big),
           Feat(table, rand_ids(rng, n, 5000), splits_of(lens), rng.uniform(0, 1, size=n).astype(f32), "mean"),
           Feat(table, rand_ids(rng, 1, 5000), np.array([0, 1], np.int64), None, "sqrtn"),
           Feat(table, rand_ids(rng, 7, 5000), splits_of([3, 0, 4]), None, "sum", 2)]
  run_ops(tfrs, feats, launches=(1, 1))


@pytest.mark.parametrize("bags", [0, 5])
def test_all_features_empty(tfrs, bags):
  """Every feature has n = 0: zero bags launch nothing; B empty bags launch the forward once (zero rows, D = 0) and
  the backward not at all."""
  rng = np.random.default_rng(23)
  t = rng.standard_normal((10, 8)).astype(f32)
  e = np.zeros(0, np.int64)
  sp = np.zeros(bags + 1, np.int64)
  feats = [Feat(t, e, sp, None, "mean"), Feat(t, e.astype(np.int32), sp, np.zeros(0, f32), "sqrtn"),
           Feat(t, e, sp, None, "sum", 3)]
  if bags == 0:
    feats.append(Feat(t, e))
  run_ops(tfrs, feats, launches=(1 if bags else 0, 0))


# ---- 9. strided outputs and gradients through ops ----------------------------------------------------------------------------
def test_shared_wide_output(tfrs):
  """Features writing disjoint column ranges of one [B, 160] output (ld > dim, col_off > 0, float4 and scalar pieces);
  every other column keeps its NaN bits; the backward reads column slices of one wider gradient."""
  rng = np.random.default_rng(24)
  lens = every_length(rng)
  sp, n = splits_of(lens), int(lens.sum())
  B, LD = len(lens), 160
  layout = [(8, 4, "sum"), (12, 16, "mean"), (3, 29, "sqrtn"), (64, 32, "mean"), (5, 100, "sum"), (20, 136, "sqrtn")]
  feats = []
  for d, _, c in layout:
    t = rng.standard_normal((31, d)).astype(f32)
    feats.append(Feat(t, rand_ids(rng, n, 31), sp, rng.uniform(-1, 2, size=n).astype(f32), c))
  wide = filled((B, LD))
  g = dev(rng.standard_normal((B, LD + 8)).astype(f32))[:, 4:4 + LD]
  run_ops(tfrs, feats, outs=[wide] * len(feats), col_offs=[c for _, c, _ in layout], grads=[g] * len(feats))
  untouched = np.ones(LD, bool)
  for d, c, _ in layout:
    untouched[c:c + d] = False
  assert (wide.cpu().numpy()[:, untouched].view(np.uint32) == NAN_FILL).all()


def test_gradient_column_slices(tfrs):
  """Sequence and dense features reading their gradients from column slices of wider gradients (ld > dim, col_off > 0,
  one of them 4 bytes off its alignment) into rows of one shared buffer."""
  rng = np.random.default_rng(25)
  t = rng.standard_normal((40, 12)).astype(f32)
  lens = every_length(rng)
  n = int(lens.sum())
  feats = [Feat(t, rand_ids(rng, n, 40), splits_of(lens), rng.uniform(-1, 1, size=n).astype(f32), "mean", 3),
           Feat(t, rand_ids(rng, 50, 40))]
  wide = [dev(rng.standard_normal((out_rows(f), 40)).astype(f32)) for f in feats]
  grads = [wide[0], dev(rng.standard_normal((50, 48)).astype(f32))[:, 5:45]]     # 4 bytes off, ld 48
  outs = [filled((out_rows(f), 40)) for f in feats]
  buf = filled((n + 50, 12))
  run_ops(tfrs, feats, outs=outs, col_offs=[8, 20], grads=grads, grad_rows=[buf[:n], buf[n:]])


def _bad_views(rows, dim):
  """(name, view) pairs that must be refused for a feature of `rows` output rows and `dim` columns at col_off 0."""
  flat = torch.zeros(rows * (dim + 8) + 64, device="cuda")
  return [("expanded (stride 0)", torch.zeros(1, dim, device="cuda").expand(rows, dim)),
          ("columns past the width", flat[:rows * (dim + 8)].view(rows, dim + 8)[:, :dim - 4]),
          ("overlapping rows", flat.as_strided((rows, dim), (dim - 4, 1)))]


def test_bad_views_raise_before_launch(tfrs):
  """Outputs and gradients whose columns leave the view, or whose rows overlap, raise ValueError in K11 and K8 before
  anything is launched."""
  ops = tfrs.ops
  rng = np.random.default_rng(26)
  dim, B = 16, 6
  t = dev(rng.standard_normal((20, dim)).astype(f32))
  v = dev(rng.integers(0, 20, size=12))
  sp = dev(splits_of([2, 2, 2, 0, 3, 3]))
  good = ops.BagFeature(t, v, torch.zeros(B, dim, device="cuda"), sp, None, "mean", 0, 0, None,
                        torch.zeros(B, device="cuda"))
  rows = torch.zeros(12, dim, device="cuda")
  ue_t = dev(rng.standard_normal((20, dim)).astype(f32))
  ue_in = [ops.LookupInput(v, None, sp, "mean")]
  ue_ids = torch.zeros(12, dtype=torch.int64, device="cuda")
  torch.cuda.synchronize()
  n0 = ops.launch_count()
  for name, bad in _bad_views(B, dim):
    with pytest.raises(ValueError, match="embedding_bag"):
      ops.embedding_bag([good._replace(out=bad)])
    with pytest.raises(ValueError, match="embedding_bag_bwd"):
      ops.embedding_bag_bwd([good], [bad], [rows])
    with pytest.raises(ValueError, match="unified_lookup"):
      ops.unified_lookup(ue_in, [ops.LookupSlot(0, ue_t, (1, 2), bad, 0, ue_ids)])
    with pytest.raises(ValueError, match="unified_lookup"):
      ops.unified_lookup_bwd(ue_in, [ops.LookupSlot(0, ue_t, (1, 2), good.out, 0, ue_ids)], [bad], [rows])
  wide = torch.zeros(B, dim + 8, device="cuda")
  for off in (12, -4):                                   # columns [off, off + dim) outside a view with a large ld
    with pytest.raises(ValueError, match="columns"):
      ops.embedding_bag([good._replace(out=wide[:, :dim + 4], col_off=off)])
    with pytest.raises(ValueError, match="columns"):
      ops.unified_lookup(ue_in, [ops.LookupSlot(0, ue_t, (1, 2), wide[:, :dim + 4], off, ue_ids)])
  with pytest.raises(ValueError, match="row_splits"):
    ops.embedding_bag([good._replace(row_splits=dev(splits_of([2, 2, 2, 0, 3, 3] * 2))[::2])])
  with pytest.raises(ValueError, match="row_splits"):
    ops.unified_lookup([ops.LookupInput(v, None, dev(splits_of([2, 2, 2, 0, 3, 3] * 2))[::2], "mean")],
                       [ops.LookupSlot(0, ue_t, (1, 2), good.out, 0, ue_ids)])
  assert ops.launch_count() == n0
  # a one-row view may have any row stride; the good feature runs
  one = good._replace(values=v[:2], row_splits=dev(np.array([0, 2], np.int64)), out=wide[:1, 4:4 + dim],
                      denom=torch.zeros(1, device="cuda"))
  ops.embedding_bag([one, good])
  assert ops.launch_count() == n0 + 1


# ---- 10. through the layer -------------------------------------------------------------------------------------------------
def _layer_check(tfrs, feats, inputs, weights, grads_of=None, launches=None, seed=0):
  """TPUEmbedding over `feats` (one FeatureConfig per feature, tables shared by identity of the host table) fed
  `inputs` / `weights`; outputs and each table's (ids, rows) pair against the reference.  `grads_of(outs)` gives the
  tensors to call backward on and their gradients (default: the outputs and random gradients)."""
  T, F = tfrs.layers.embedding.TableConfig, tfrs.layers.embedding.FeatureConfig
  host_tables, cfgs = {}, {}
  fcs = []
  for f in feats:
    key = (id(f.table), f.combiner)
    if key not in cfgs:
      init = (lambda a: lambda shape, device: torch.from_numpy(a).to(device))(f.table)
      cfgs[key] = T(f.table.shape[0], f.table.shape[1], initializer=init, combiner=f.combiner)
      host_tables[key] = f.table
    fcs.append(F(cfgs[key], max_sequence_length=f.L))
  layer = tfrs.layers.embedding.TPUEmbedding(fcs)
  torch.cuda.synchronize()
  n0 = tfrs.ops.launch_count()
  outs = layer(inputs, weights)
  n1 = tfrs.ops.launch_count()
  for k, (f, o) in enumerate(zip(feats, outs)):
    r, _ = ref_forward(f)
    shape = (tuple(np.shape(f.ids)) + (f.table.shape[1],) if f.splits is None else
             (len(f.splits) - 1, f.L, f.table.shape[1]) if f.L else (len(f.splits) - 1, f.table.shape[1]))
    same(o, r.reshape(shape), f"layer output {k}")
  rng = np.random.default_rng(seed)
  if grads_of is None:
    tensors, gs = outs, [dev(rng.standard_normal(tuple(o.shape)).astype(f32)) for o in outs]
    dl_dout = [g.cpu().numpy() for g in gs]
  else:
    proxies = [o.detach().clone().requires_grad_() for o in outs]
    pt, pg = grads_of(proxies, rng)
    torch.autograd.backward(pt, pg)
    dl_dout = [p.grad.cpu().numpy() if p.grad is not None else np.zeros(tuple(p.shape), f32) for p in proxies]
    tensors, gs = grads_of(outs, np.random.default_rng(seed))
  n2 = tfrs.ops.launch_count()
  torch.autograd.backward(tensors, gs)
  n3 = tfrs.ops.launch_count()
  exp = {}
  for f, fc, g in zip(feats, fcs, dl_dout):
    exp.setdefault(id(fc.table), []).append((f.ids.astype(np.int64).reshape(-1),
                                             ref_backward(f, g.reshape(-1, f.table.shape[1]))))
  for c, tab in layer.embedding_tables.items():
    pairs = tab.pop_sparse_grads()
    assert len(pairs) == 1
    same(pairs[0][0], np.concatenate([i for i, _ in exp[id(c)]]), "ids of a table's pair")
    same(pairs[0][1], np.concatenate([r for _, r in exp[id(c)]]), "rows of a table's pair")
  if launches is not None:
    assert (n1 - n0, n3 - n2) == launches
  return layer, outs


def _to_sparse(ids, sp, dtype):
  B = len(sp) - 1
  rows = np.repeat(np.arange(B), np.diff(sp))
  cols = np.arange(ids.size) - sp[rows]
  idx = torch.from_numpy(np.stack([rows, cols])).cuda()
  width = max(int(np.diff(sp).max(initial=0)), 1)
  return torch.sparse_coo_tensor(idx, torch.from_numpy(ids).to(dtype).cuda(), (B, width)).coalesce()


def test_layer_split_forms(tfrs):
  """Row splits as NumPy arrays (sharing one upload at non-zero offsets), as CUDA tensors and from sparse COO inputs,
  with empty-bag runs, in one call."""
  rng = np.random.default_rng(27)
  t = rng.standard_normal((30, 8)).astype(f32)
  t2 = rng.standard_normal((19, 5)).astype(f32)
  feats, inputs, weights = [], [], []
  for k, form in enumerate(["numpy", "numpy", "cuda", "sparse", "numpy", "dense"]):
    lens = every_length(rng)
    sp, n = splits_of(lens), int(lens.sum())
    tab = t if k % 2 == 0 else t2
    ids = rand_ids(rng, n, tab.shape[0], np.int32 if form == "sparse" else np.int64)
    w = rng.uniform(0, 2, size=n).astype(f32)
    if form == "dense":
      feats.append(Feat(tab, ids[:40].reshape(8, 5)))
      inputs.append(dev(ids[:40].reshape(8, 5)))
      weights.append(None)
      continue
    feats.append(Feat(tab, ids, sp, w, ("mean", "sqrtn", "sum")[k % 3], 3 if k == 4 else 0))
    if form == "sparse":
      inputs.append(_to_sparse(ids, sp, torch.int32))
      weights.append(torch.sparse_coo_tensor(inputs[-1].indices(), dev(w), inputs[-1].shape))
    else:
      inputs.append((dev(ids), sp if form == "numpy" else dev(sp)))
      weights.append(dev(w))
  layer, outs = _layer_check(tfrs, feats, inputs, weights, launches=(1, 1))
  node = outs[0].grad_fn
  splits = [f.row_splits for f in node.feats]
  base = splits[0].untyped_storage().data_ptr()
  assert [s.untyped_storage().data_ptr() == base for s in splits[:5]] == [True, True, False, False, True]
  assert splits[1].storage_offset() > 0 and splits[4].storage_offset() > splits[1].storage_offset()


def test_layer_view_gradients(tfrs):
  """Outputs transposed, sliced and expanded before the loss: the layer's backward takes each gradient as it comes."""
  rng = np.random.default_rng(28)
  t = rng.standard_normal((25, 12)).astype(f32)
  lens = every_length(rng)
  sp, n = splits_of(lens), int(lens.sum())
  ids = rand_ids(rng, n, 25)
  w = rng.uniform(-1, 2, size=n).astype(f32)
  feats = [Feat(t, ids, sp, w, "sqrtn"), Feat(t, ids, sp, w, "mean", 4), Feat(t, ids[:30].reshape(10, 3))]
  inputs = [(dev(ids), sp), (dev(ids), dev(sp)), dev(ids[:30].reshape(10, 3))]

  def grads_of(outs, r):
    w0 = dev(r.standard_normal((12, len(lens))).astype(f32))
    w1 = dev(r.standard_normal((3,) + tuple(outs[1].shape)).astype(f32))
    w2 = dev(r.standard_normal((10, 3, 12)).astype(f32))
    loss = ((outs[0].t()[::2] * w0[::2]).sum() + (outs[1][:, 1:3].expand(3, -1, -1, -1) * w1[:, :, 1:3]).sum() +
            (outs[2][:, :, 2:9] * w2[:, :, 2:9]).sum())
    return [loss], [torch.ones((), device="cuda")]

  _layer_check(tfrs, feats, inputs, [dev(w), dev(w), None], grads_of=grads_of)
  torch.cuda.synchronize()


@pytest.mark.parametrize("count", [128, 129, 257])
def test_layer_tables_across_groups(tfrs, count):
  """Features of three shared tables across the 128-feature boundaries: each table's (ids, rows) pair stays in
  feature order; one launch each way per group."""
  rng = np.random.default_rng(100 + count)
  tables = [rng.standard_normal((r, d)).astype(f32) for r, d in ((17, 4), (9, 3), (23, 8))]
  feats = _mixed_features(rng, count, tables)
  inputs, weights = [], []
  for f in feats:
    if f.splits is None:
      inputs.append(dev(f.ids))
      weights.append(None)
    else:
      inputs.append((dev(f.ids), f.splits))
      weights.append(dev(f.weights))
  g = -(-count // BG_MAX_FEATURES)
  _layer_check(tfrs, feats, inputs, weights, launches=(g, g), seed=count)


# ---- 11. argument errors -----------------------------------------------------------------------------------------------------
def test_argument_errors(tfrs):
  """Each argument check of bg_check (through the C entry points) and of the Python wrappers raises before any launch."""
  ops = tfrs.ops
  rng = np.random.default_rng(29)
  dim, B = 8, 4
  t = dev(rng.standard_normal((20, dim)).astype(f32))
  v = dev(rng.integers(0, 20, size=9))
  sp = dev(splits_of([2, 3, 0, 4]))
  good = ops.BagFeature(t, v, torch.zeros(B, dim, device="cuda"), sp, dev(np.ones(9, f32)), "mean", 0, 0,
                        torch.zeros(9, dtype=torch.int64, device="cuda"), torch.zeros(B, device="cuda"))
  g = torch.zeros(B, dim, device="cuda")
  r = torch.zeros(9, dim, device="cuda")

  def c_call(bwd, **change):
    cs = ops._bag_structs([good], [g if bwd else good.out], "test")
    cs[0].out = good.out.data_ptr()
    if bwd:
      cs[0].grad, cs[0].grad_rows = g.data_ptr(), r.data_ptr()
    for k, x in change.items():
      setattr(cs[0], k, x)
    fn = ops.lib().tfrs_embedding_bag_bwd_f32 if bwd else ops.lib().tfrs_embedding_bag_fwd_f32
    ops.check(fn(cs, 1, ops.stream()), "embedding_bag")

  torch.cuda.synchronize()
  n0 = ops.launch_count()
  with pytest.raises(ValueError, match="empty call"):
    ops.check(ops.lib().tfrs_embedding_bag_fwd_f32(None, 0, ops.stream()), "embedding_bag")
  with pytest.raises(ValueError, match="empty call"):
    ops.check(ops.lib().tfrs_embedding_bag_bwd_f32((ops._BagFeature * 1)(), 0, ops.stream()), "embedding_bag")
  c_errors = [(dict(dim=0), "NULL table"), (dict(rows=0), "NULL table"), (dict(table=None), "NULL table"),
              (dict(kind=2), "kind"), (dict(n=-1), "bad n"), (dict(n=1 << 40), "bad n"), (dict(values=None), "bad n"),
              (dict(max_seq_len=-1), "max_seq_len"), (dict(row_splits=None), "dense feature"),
              (dict(n_bags=-1), "combiner"), (dict(combiner=3), "combiner"), (dict(combiner=-1), "combiner"),
              (dict(n_bags=0), "no bag"), (dict(col_off=-4), "outside ld"), (dict(col_off=4), "outside ld"),
              (dict(ld=dim - 1), "outside ld")]
  for bwd in (False, True):
    for change, msg in c_errors:
      with pytest.raises(ValueError, match=msg):
        c_call(bwd, **change)
  with pytest.raises(ValueError, match="NULL out"):
    c_call(False, out=None)
  for change in (dict(grad=None), dict(grad_rows=None)):
    with pytest.raises(ValueError, match="NULL grad"):
      c_call(True, **change)
  with pytest.raises(ValueError, match="denominators"):
    c_call(True, denom=None)
  with pytest.raises(ValueError, match="dense feature"):                 # a dense feature with a max_seq_len
    c_call(False, row_splits=None, weights=None, max_seq_len=2)
  py_errors = [dict(table=t.t()), dict(table=t.double()), dict(table=t[None]), dict(values=v.view(3, 3).t()),
               dict(weights=dev(np.ones(8, f32))), dict(weights=dev(np.ones(9, np.float64))),
               dict(weights=dev(np.ones(18, f32))[::2]), dict(out=torch.zeros(B + 1, dim, device="cuda")),
               dict(out=torch.zeros(B, dim, device="cuda", dtype=torch.float64)),
               dict(out=torch.zeros(dim, B, device="cuda").t()), dict(out=torch.zeros(B, dim - 1, device="cuda")),
               dict(col_off=1), dict(ids=torch.zeros(8, dtype=torch.int64, device="cuda")),
               dict(ids=torch.zeros(9, dtype=torch.int32, device="cuda")),
               dict(denom=torch.zeros(B + 1, device="cuda")), dict(denom=torch.zeros(B, device="cuda").double()),
               dict(row_splits=dev(splits_of([2, 3, 0, 4, 0]))[::2])]
  for change in py_errors:
    with pytest.raises(ValueError):
      ops.embedding_bag([good._replace(**change)])
  for change in (dict(row_splits=sp.int()), dict(row_splits=sp.view(1, -1)), dict(row_splits=sp[:0])):
    with pytest.raises(TypeError):
      ops.embedding_bag([good._replace(**change)])
  for change in (dict(table=t.cpu()), dict(values=v.cpu()), dict(weights=good.weights.cpu()), dict(ids=good.ids.cpu()),
                 dict(denom=good.denom.cpu()), dict(row_splits=sp.cpu()), dict(out=good.out.cpu())):
    with pytest.raises((ValueError, TypeError, RuntimeError)):       # require_cuda raises RuntimeError
      ops.embedding_bag([good._replace(**change)])
  for bad in ([[g, g], [r]], [[g], [r, r]], [[g], [r[:8]]], [[g], [r.t().contiguous().t()]], [[g], [r.double()]],
              [[g], [r.cpu()]], [[g[:3]], [r]]):
    with pytest.raises((ValueError, TypeError, RuntimeError)):
      ops.embedding_bag_bwd([good], *bad)
  assert ops.launch_count() == n0
  ops.embedding_bag([good])
  ops.embedding_bag_bwd([good], [g], [r])
  assert ops.launch_count() == n0 + 2
