"""The K19 / K20 recurrence kernels' tile and shared-memory plan restated from csrc/rnn.cuh (rnn_tile, rnn_smem), and
the edge cases generated from it for tests/test_gpu_rnn_edges.py, which tests/test_rnn_plan_host.py checks reach every
instance, slice edge, batch, length, mask kind, pattern and value the plan makes interesting.

Each Case names a cell, u, B, T, a mask kind (None, "bool", "int32", "int64") and pattern, and which nullable inputs
and outputs the call passes; `inputs(case)` makes its float32 data."""
import dataclasses
import math

import numpy as np

THREADS, PAIRS, SMEM_MAX, SLICE_BYTES = 256, 8, 227 * 1024, 64 * 1024   # RNN_* of csrc/rnn.cuh
MAX_UNITS = 2048
NG = {"gru": 3, "lstm": 4}
CELLS = ("gru", "lstm")
DIRS = ("fwd", "bwd")
UJS = (1, 2, 4, 8)
MASK_KINDS = (None, "bool", "int32", "int64")
PATTERNS = ("random", "leading", "trailing", "edges")
INT32_MIN, INT64_MIN = -2 ** 31, -2 ** 63
NONZERO = {"bool": (1,), "int32": (1, 2, -1, INT32_MIN), "int64": (1, 2 ** 32, INT64_MIN, -1)}
DTYPES = {"bool": np.bool_, "int32": np.int32, "int64": np.int64}
WAVE_CTAS = 132 * 8             # more CTAs than an H100 can hold at once (132 SMs, at most 2048 / 256 CTAs each)


@dataclasses.dataclass(frozen=True)
class Tile:
  jt: int
  g: int
  uj: int
  rj: int
  rows: int


def tile(u):
  jt = 32
  while jt < u and jt < THREADS:
    jt *= 2
  g = THREADS // jt
  uj = 1
  while uj * jt < u:
    uj *= 2
  rj = PAIRS // uj
  return Tile(jt, g, uj, rj, g * rj)


def smem(fixed_floats, rows_total, per):
  """(slice rows, bytes) of rnn_smem."""
  fixed, whole = fixed_floats * 4, rows_total * per * 4
  if fixed + whole <= SMEM_MAX:
    return rows_total, fixed + whole
  s = max(1, SLICE_BYTES // (per * 4))
  return s, fixed + s * per * 4


@dataclasses.dataclass(frozen=True)
class Plan:
  tile: Tile
  slice_rows: int        # ks (forward: rows of U) or cs (reverse: columns of U, rows of U^T)
  total: int             # u or NG u
  resident: bool

  @property
  def last(self):
    """rows (columns) in the last slice"""
    return self.total - (math.ceil(self.total / self.slice_rows) - 1) * self.slice_rows


def plan(cell, direction, u):
  t, ng = tile(u), NG[cell]
  if direction == "fwd":
    ks, _ = smem(2 * t.rows * u, u, ng * u)
    return Plan(t, ks, u, ks >= u)
  cs, _ = smem(2 * t.rows * ng * u, ng * u, u + 1)
  return Plan(t, cs, ng * u, cs >= ng * u)


def units_of(uj):
  return [u for u in range(1, MAX_UNITS + 1) if tile(u).uj == uj]


def resident_edges(cell, direction):
  """every u after which the weights stop or start being resident"""
  return [u for u in range(1, MAX_UNITS) if plan(cell, direction, u).resident != plan(cell, direction, u + 1).resident]


def slice_edge_units(cell, direction, uj):
  """(u whose last slice is the shortest, u whose slices divide exactly) among the streamed u of the instance, or None
  where no u of the instance streams.  The shortest is one row (column) everywhere but LSTM's reverse at UJ = 1, whose
  4u columns and even slice widths leave at least 4."""
  us = [u for u in units_of(uj) if not plan(cell, direction, u).resident]
  if not us:
    return None
  shortest = min(plan(cell, direction, u).last for u in us)
  one = next(u for u in us if plan(cell, direction, u).last == shortest)
  full = next(u for u in us if plan(cell, direction, u).last == plan(cell, direction, u).slice_rows)
  return one, full


@dataclasses.dataclass(frozen=True)
class Case:
  name: str
  cell: str
  u: int
  B: int
  T: int
  kind: object = None            # mask element type
  pattern: str = "random"
  opts: int = 0                  # index into OPTS[cell]
  seed: int = 0
  contractive: bool = False      # U with every row's |U| sum below 1 (long T)


# the nullable inputs and outputs of a call: h0 / c0 / b_r / out_seq in the forward, the upstream gradients and the
# initial-state gradients in the reverse
OPTS = {
    "gru": [dict(h0=1, br=1, seq=1, g_seq=1, g_last=1, dh0=1),
            dict(h0=0, br=0, seq=1, g_seq=1, g_last=0, dh0=1),
            dict(h0=1, br=0, seq=0, g_seq=0, g_last=1, dh0=1),
            dict(h0=0, br=1, seq=1, g_seq=1, g_last=0, dh0=0)],
    "lstm": [dict(h0=1, c0=1, seq=1, g_seq=1, g_h=1, g_c=1, dh0=1, dc0=1),
             dict(h0=0, c0=0, seq=1, g_seq=1, g_h=0, g_c=0, dh0=1, dc0=1),
             dict(h0=1, c0=0, seq=0, g_seq=0, g_h=1, g_c=0, dh0=0, dc0=1),
             dict(h0=0, c0=1, seq=1, g_seq=0, g_h=0, g_c=1, dh0=1, dc0=0)],
}
REP_U = {1: 33, 2: 300, 4: 600, 8: 1100}      # one u per instance, away from its edges


def _cases():
  out, n = [], 0

  def add(name, cell, u, B, T, kind=None, pattern="random"):
    nonlocal n
    # beyond ten steps, U contractive and every upstream gradient given, so that the carried bound stays meaningful
    long_ = T > 10
    out.append(Case(name, cell, u, B, T, kind, pattern if kind else "random", 0 if long_ else n % 4, 1000 + n, long_))
    n += 1

  for cell in CELLS:
    # every instance: (UJ, mask kind), at B = R + 1 (a partial last CTA)
    for uj in UJS:
      for m, kind in enumerate(MASK_KINDS):
        u = REP_U[uj] + m
        add(f"{cell}-uj{uj}-{kind}", cell, u, tile(u).rows + 1, 3 if uj > 1 else 5, kind, PATTERNS[(uj + m) % 4])
    # resident / streamed flips at UJ = 1, both directions
    for d in DIRS:
      for e in resident_edges(cell, d):
        for u in (e, e + 1):
          add(f"{cell}-{d}-edge-u{u}", cell, u, tile(u).rows + 1, 3, MASK_KINDS[u % 4], "edges")
    # last slice of one row (column), and slices that divide exactly, in every streamed instance
    for d in DIRS:
      for uj in UJS:
        se = slice_edge_units(cell, d, uj)
        for what, u in zip(("one", "exact"), se or ()):
          add(f"{cell}-{d}-uj{uj}-slice-{what}-u{u}", cell, u, 2 if uj > 1 else tile(u).rows - 1, 2,
              MASK_KINDS[(u + uj) % 4], PATTERNS[u % 4])
    # batch: 1, R - 1, R, R + 1 at two instances, and more than one wave of CTAs
    for u in (33, 257):
      R = tile(u).rows
      for B in sorted({1, R - 1, R, R + 1} - {0}):
        add(f"{cell}-u{u}-B{B}", cell, u, B, 3, "int32" if B % 2 else "bool", "edges")
    R = tile(8).rows
    add(f"{cell}-waves", cell, 8, R * WAVE_CTAS + 3, 2, "int64", "random")
    # lengths: 1, 2, 3, odd >= 65, and about 1000 steps at small u
    for T in (1, 2, 3, 65, 129):
      add(f"{cell}-T{T}", cell, 40, 33, T, "bool" if T > 1 else None, "edges")
    add(f"{cell}-T1001", cell, 8, 65, 1001, "int32", "random")
    add(f"{cell}-T999-u130", cell, 130, 9, 999, None)
  return out


CASES = _cases()


def mask_values(kind, keep, rng):
  """keep [B, T] bool -> the kind's array, nonzero entries drawn from NONZERO[kind] (all count as kept)"""
  if kind is None:
    return None
  if kind == "bool":
    return keep.copy()
  vals = np.array(NONZERO[kind], DTYPES[kind])
  return np.where(keep, vals[rng.randint(0, len(vals), size=keep.shape)], 0).astype(DTYPES[kind])


def keep_pattern(pattern, B, T, rng):
  if pattern == "random":
    k = rng.rand(B, T) < 0.6
  elif pattern == "leading":              # the first steps of each row masked
    k = np.arange(T)[None] >= rng.randint(0, T + 1, size=(B, 1))
  elif pattern == "trailing":
    k = np.arange(T)[None] < rng.randint(0, T + 1, size=(B, 1))
  else:                                   # "edges": a fully masked row, rows masked only at t = 0 / only at T - 1
    k = rng.rand(B, T) < 0.7
    k[0::4] = False
    k[1::4] = True
    k[1::4, 0] = False
    k[2::4] = True
    k[2::4, T - 1] = False
  return k


def inputs(case, rows=None):
  """float32 data of a case: dict of gx [B, T, NG u], U, b_r (GRU), h0, c0 (LSTM), the upstream gradients, keep [B, T]
  and the mask array in the case's kind (None where the option is off).  rows: only these batch rows (a row's data
  do not depend on B)."""
  rng = np.random.RandomState(case.seed)
  cell, u, T = case.cell, case.u, case.T
  ng = NG[cell]
  if case.contractive:      # row sums of |U| about 0.8
    U = rng.uniform(-1, 1, size=(u, ng * u)) * (1.6 / (ng * u))
  else:                     # column sums of |U| about 1, so that the forward's carried bound does not grow with u
    U = rng.normal(size=(u, ng * u)) * (1.2 / u)
  o = OPTS[cell][case.opts]
  B = case.B
  rows = np.arange(B) if rows is None else np.asarray(rows)
  d = {"U": U.astype(np.float32)}
  d["b_r"] = (rng.normal(size=ng * u) * 0.2).astype(np.float32) if cell == "gru" and o["br"] else None
  keep_all = keep_pattern(case.pattern, B, T, rng) if case.kind else np.ones((B, T), bool)
  keep = keep_all[rows]
  d["keep"] = keep
  d["mask"] = mask_values(case.kind, keep, np.random.RandomState(case.seed + 1)) if case.kind else None

  def per_row(shape, scale, salt):
    """row b's data from its own seed, so a subset of rows is the same data"""
    return np.stack([np.random.RandomState([case.seed, salt, int(b)]).normal(size=shape) * scale for b in rows]
                    ).astype(np.float32) if len(rows) else np.zeros((0,) + shape, np.float32)

  d["gx"] = per_row((T, ng * u), 1.0, 1)
  d["h0"] = per_row((u,), 0.5, 2) if o["h0"] else None
  d["c0"] = per_row((u,), 1.0, 3) if cell == "lstm" and o["c0"] else None
  d["g_seq"] = per_row((T, u), 1.0, 4) if o["g_seq"] else None
  last = "g_last" if cell == "gru" else "g_h"
  d[last] = per_row((u,), 1.0, 5) if o[last] else None
  d["g_c"] = per_row((u,), 1.0, 6) if cell == "lstm" and o["g_c"] else None
  return d
