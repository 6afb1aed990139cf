"""Edge cases of K4's id grouping and run summing (csrc/adagrad.cu, csrc/adagrad.cuh), through every sparse optimizer that
uses them: SGD (sgd.cu), Adagrad (adagrad.cu's fused ag_apply / ag_apply_long), ClippyAdagrad, Adam and FTRL (the
ag_sum_runs / ag_sum_runs_long templates), and TreeAH's leaf grouping (tree_ah.cu, the bitonic branch ag_sort).

The code under test turns a batch's (id, gradient row) pairs into one update per touched row: keys (id << 24 | position)
are grouped by id with positions ascending -- a bucketed rank sort up to AG_RANK_MAX ids, a bitonic sort in AG_TILE-key
shared-memory tiles plus global strides beyond -- and each run of equal ids is summed in order of occurrence, the first
member starting the sum.  A warp sums runs of up to AG_LONG members (run end found with 32-slot ballots, 8 rows in flight
per step); one CTA per longer run finds the end with AL_THREADS-key windows and stages tile_rows(d) gradient rows at a
time through 64 KB of shared memory (float4 loads when d % 4 == 0 and the rows are 16-byte aligned).

Every GPU result is compared bit for bit, on every state array and on ClippyAdagrad's clipping factor, with a CPU
reference of the same step (two NaNs count as equal whatever their payloads):
  SGD          `_sgd_ref`, a vectorised restatement of embedding_bag_oracle.sgd_sparse (checked against it on the CPU)
  Adagrad      oracle.orc.sparse_adagrad; past ORC_MAX_N ids `_adagrad_ref`, checked against it on the CPU
  ClippyAdagrad, Adam, FTRL   tests/clippy_oracle.py, adam_oracle.py, ftrl_oracle.py
FTRL's pow mode rounds a float64 pow to fp32 once, on the GPU and in NumPy; where the two libraries round that pow to
different floats the element is accepted only if the reference reproduces the GPU's bits with its power terms moved by
one ulp (`_ftrl_pow_explained`).  The gradient sum itself is still held bit for bit.

The case families, the constants they are built around (read back from the sources by a CPU test, so that a change to a
constant fails the case set instead of leaving it stale), and the order-of-summation self-test are in DESIGN.md
section 2.  The GPU tests are marked one by one; the case-set checks and self-tests run without a GPU.
"""
import functools
import os
import re

import numpy as np
import pytest
import torch

import adam_oracle as ao
import clippy_oracle as co
import embedding_bag_oracle as ebo
import ftrl_oracle as fo
from oracle import oracle as orc

gpu = pytest.mark.gpu
F32 = np.float32

# csrc/adagrad.cu and csrc/adagrad.cuh (test_constants_and_shared_checks_match_the_sources reads them back)
AG_RANK_MAX = 16384      # bucketed rank sort up to here, bitonic sort beyond
AG_TILE = 8192           # keys per shared-memory tile of the bitonic sort
AB_BUCKETS = 256
AB_SPLIT = 8             # slices per bucket in ag_bucket_rank
AG_LONG = 64             # longest run the warp kernels sum
AL_THREADS = 256         # threads of the CTA-per-run kernels: run end found in windows of this many keys
AL_ROWS = 256            # most gradient rows staged per tile
AL_SMEM = 64 * 1024      # shared-memory staging budget of the long-run kernels
H100_SMS = 132           # the long-run kernels launch one CTA per SM and stride over the runs
MAX_N = 1 << 24          # n must be below 2^24: the position takes the key's low 24 bits

INT32_MIN, INT32_MAX = -2 ** 31, 2 ** 31 - 1
INT64_MIN, INT64_MAX = -2 ** 63, 2 ** 63 - 1
IDTS = (torch.int32, torch.int64)
ORC_MAX_N = 40000        # orc.sparse_adagrad is O(n^2) in the ids; past this the vectorised restatement is used

VARIANTS = {
    "sgd": ("sgd", dict(lr=0.3)),
    "adagrad_eps_inside": ("adagrad", dict(lr=0.1, eps=1e-7, eps_inside_sqrt=True)),
    "adagrad_eps_outside": ("adagrad", dict(lr=0.1, eps=1e-3, eps_inside_sqrt=False)),
    # thresholds small enough that the factor is well below 1 whenever a gradient is not zero
    "clippy_flags0": ("clippy", dict(lr=0.1, eps=1e-7, var_rel=1e-3, acc_rel=1e-4, abs_thr=1e-6, clip=False, standard=False)),
    "clippy_flags2": ("clippy", dict(lr=0.1, eps=1e-7, var_rel=1e-3, acc_rel=1e-4, abs_thr=1e-6, clip=False, standard=True)),
    "adam": ("adam", dict(lr=0.01, t=3, beta_1=0.9, beta_2=0.999, epsilon=1e-7, lazy=False)),
    "adam_lazy": ("adam", dict(lr=0.01, t=3, beta_1=0.9, beta_2=0.999, epsilon=1e-7, lazy=True)),
    "ftrl_sqrt_shrink": ("ftrl", dict(lr=0.05, lr_power=-0.5, l1=0.02, l2=0.01, l2_shrinkage=0.3, beta=0.5)),
    "ftrl_pow": ("ftrl", dict(lr=0.05, lr_power=-0.75, l1=0.02, l2=0.01)),
}
ALL = tuple(VARIANTS)
WS_SLOT = {"sgd": "sgd", "adagrad": "adagrad", "clippy": "clippy", "adam": "adam", "ftrl": "ftrl"}


@pytest.fixture(scope="module")
def ops():
  from recommenders_b200 import ops as o
  return o


# ------------------------------------------------------------------------------------------------
# The kernels' rules, restated
# ------------------------------------------------------------------------------------------------
def tile_rows(d):
  """Gradient rows the long-run kernels stage per tile at width d."""
  return max(1, min(AL_ROWS, AL_SMEM // (4 * d)))


def padded(n):
  """P, the bitonic sort's padded size."""
  p = 1
  while p < max(n, 2):
    p <<= 1
  return p


def ag_bucket(ids):
  """ag_bucket of the keys of in-range ids (0 <= id < 2^40): ((id & 0xFFFFFFFF) ^ (id >> 32)) * 0x9E3779B1 mod 2^32 >> 24."""
  x = np.asarray(ids, np.int64).astype(np.uint64)
  m = np.uint64(0xFFFFFFFF)
  h = ((x & m) ^ (x >> np.uint64(32))) & m
  return ((h * np.uint64(0x9E3779B1)) & m) >> np.uint64(24)


# ------------------------------------------------------------------------------------------------
# References
# ------------------------------------------------------------------------------------------------
def _runs(ids, rows):
  """Runs of equal in-range ids, longest first: (ids, member positions in order of occurrence as `order[start + k]`,
  starts, counts).  The runs still going at member k are a prefix, so a step over them costs only their number."""
  ids = np.asarray(ids, np.int64).reshape(-1)
  pos = np.flatnonzero((ids >= 0) & (ids < rows))
  order = pos[np.argsort(ids[pos], kind="stable")]
  sid = ids[order]
  starts = np.flatnonzero(np.r_[True, sid[1:] != sid[:-1]]) if sid.size else np.zeros(0, np.int64)
  counts = np.diff(np.r_[starts, sid.size]).astype(np.int64)
  by = np.argsort(-counts, kind="stable")
  return sid[starts][by], order, starts[by], counts[by]


def _active(counts, k):
  return int(np.searchsorted(-counts, -k, side="left"))     # runs with more than k members


def run_sums(ids, g, rows, mode="order"):
  """(run ids, gradient sums).  "order": in order of occurrence, the first member starting the sum (the kernels' rule);
  "zero_start": the same sum started from +0.0f; "reversed": the members added last to first."""
  heads, order, starts, counts = _runs(ids, rows)
  g = np.asarray(g, F32).reshape(np.size(ids), -1)
  member = (lambda k, a: order[starts[:a] + counts[:a] - 1 - k]) if mode == "reversed" else (lambda k, a: order[starts[:a] + k])
  sums = g[member(0, len(heads))].copy()
  if mode == "zero_start":
    sums = F32(0) + sums
  with np.errstate(all="ignore"):
    for k in range(1, int(counts[0]) if counts.size else 0):
      a = _active(counts, k)
      sums[:a] = sums[:a] + g[member(k, a)]
  return heads, sums


def _sgd_ref(table, ids, g, lr):
  """embedding_bag_oracle.sgd_sparse, vectorised: table[id] -= lr * g once per occurrence, in order of occurrence."""
  t = np.array(table, F32)
  heads, order, starts, counts = _runs(ids, t.shape[0])
  if not heads.size:
    return t
  g = np.asarray(g, F32).reshape(np.size(ids), -1)
  lr = F32(lr)
  x = t[heads]
  for k in range(int(counts[0])):
    a = _active(counts, k)
    x[:a] = x[:a] - lr * g[order[starts[:a] + k]]
  t[heads] = x
  return t


def _adagrad_ref(table, accum, ids, g, lr, eps, eps_inside_sqrt):
  """orc.sparse_adagrad's rule on run_sums: a = acc + g*g; var -= (lr*g) / sqrt(a + eps)  (or sqrt(a) + eps)."""
  t, acc = np.array(table, F32), np.array(accum, F32)
  heads, s = run_sums(ids, g, t.shape[0])
  a = acc[heads] + s * s
  with np.errstate(all="ignore"):
    den = np.sqrt(a + F32(eps)) if eps_inside_sqrt else np.sqrt(a) + F32(eps)
    t[heads] = t[heads] - (F32(lr) * s) / den
  acc[heads] = a
  return t, acc


def reference(vname, st, ids, g):
  """The reference step of one variant on copies of the state arrays: {slot: array} (+ "factor" for ClippyAdagrad)."""
  kind, kw = VARIANTS[vname]
  ids = np.asarray(ids, np.int64).reshape(-1)
  g = np.asarray(g, F32).reshape(ids.size, -1)
  with np.errstate(all="ignore"):
    if kind == "sgd":
      return {"table": _sgd_ref(st["table"], ids, g, kw["lr"])}
    if kind == "adagrad":
      if ids.size <= ORC_MAX_N:
        t, a = orc.sparse_adagrad(st["table"], st["accum"], ids, g, kw["lr"], kw["eps"], kw["eps_inside_sqrt"])
      else:
        t, a = _adagrad_ref(st["table"], st["accum"], ids, g, kw["lr"], kw["eps"], kw["eps_inside_sqrt"])
      return {"table": t, "accum": a}
    if kind == "clippy":
      t, a, f = co.clippy_adagrad_sparse(st["table"], st["accum"], ids, g, kw["lr"], kw["eps"], kw["var_rel"], kw["acc_rel"],
                                         kw["abs_thr"], kw["clip"], kw["standard"])
      return {"table": t, "accum": a, "factor": np.asarray(f, F32)}
    if kind == "adam":
      t, m, v = ao.adam_sparse(st["table"], st["m"], st["v"], ids, g, kw["lr"], kw["t"], kw["beta_1"], kw["beta_2"],
                               kw["epsilon"], kw["lazy"])
      return {"table": t, "m": m, "v": v}
    t, a, z = fo.ftrl_sparse(st["table"], st["accum"], st["linear"], ids, g, **kw)
    return {"table": t, "accum": a, "linear": z}


def _ftrl_pow_explained(st, ids, g, kw, got, want, rows_cols):
  """True when every listed element of the GPU's FTRL pow step is the reference rule's result with P(na) and P(acc)
  each moved by at most one fp32 ulp: the float64 pow of two libraries can round to neighbouring floats.  The gradient
  sum is the reference's in-order sum, so a wrong sum is not explained."""
  heads, sums = run_sums(ids, g, st["table"].shape[0])
  where = {int(h): i for i, h in enumerate(heads)}
  lr32, l1, s = F32(kw["lr"]), F32(kw["l1"]), F32(kw.get("l2_shrinkage", 0.0))
  two_l2a = F32(2) * fo.l2a(kw["l2"], kw.get("beta", 0.0), kw["lr"])
  for r, c in rows_cols:
    if int(r) not in where:
      return False
    x, a, z = st["table"][r, c], st["accum"][r, c], st["linear"][r, c]
    gg = sums[where[int(r)], c]
    na = a + gg * gg
    pn0, pa0 = fo.power(np.array([na], F32), kw["lr_power"])[0], fo.power(np.array([a], F32), kw["lr_power"])[0]
    ok = False
    for pn in (np.nextafter(pn0, F32(-np.inf)), pn0, np.nextafter(pn0, F32(np.inf))):
      for pa in (np.nextafter(pa0, F32(-np.inf)), pa0, np.nextafter(pa0, F32(np.inf))):
        with np.errstate(all="ignore"):
          gs = gg + (F32(2) * s) * x if s > 0 else gg
          lin = z + (gs - ((pn - pa) / lr32) * x)
          y = pn / lr32 + two_l2a
          var = (np.copysign(l1, lin) - lin) / y if abs(lin) > l1 else F32(0)
        if _bits(np.float32(var)) == _bits(got["table"][r, c]) and _bits(np.float32(lin)) == _bits(got["linear"][r, c]):
          ok = True
    if not ok:
      return False
  return True


def _bits(a):
  return np.asarray(a, F32).view(np.int32)


def _mismatch(got, want):
  """Elements whose bits differ (two NaNs are equal)."""
  got, want = np.asarray(got, F32), np.asarray(want, F32)
  return (_bits(got) != _bits(want)) & ~(np.isnan(got) & np.isnan(want))


def compare(vname, got, want, st=None, ids=None, g=None):
  """Error strings for every state array (and factor) whose bits differ."""
  errs = []
  bad = {k: _mismatch(got[k], want[k]) for k in want}
  if VARIANTS[vname][1].get("lr_power", -0.5) != -0.5 and st is not None and (bad["table"].any() or bad["linear"].any()):
    rc = np.argwhere(bad["table"] | bad["linear"])
    if not bad["accum"].any() and len(rc) <= 64 and _ftrl_pow_explained(st, ids, g, VARIANTS[vname][1], got, want, rc):
      bad["table"][:] = False; bad["linear"][:] = False
  for k, b in bad.items():
    if b.any():
      i = tuple(int(x) for x in np.argwhere(b)[0]) if b.ndim else ()
      gb, wb = int(_bits(got[k])[i]) & 0xFFFFFFFF, int(_bits(want[k])[i]) & 0xFFFFFFFF
      errs.append(f"{vname}.{k}: {int(b.sum())} words differ; first {i}: got {gb:#010x} want {wb:#010x}")
  return errs


# ------------------------------------------------------------------------------------------------
# State arrays, gradients, and the GPU step of each variant
# ------------------------------------------------------------------------------------------------
def init_states(vname, rows, d, seed, neg_zero_rows=()):
  """Arbitrary fp32 state arrays; accumulators positive.  On `neg_zero_rows` the weight and the slots that can be zero
  (m, v, linear) hold -0.0."""
  kind = VARIANTS[vname][0]
  rng = np.random.default_rng(seed)
  u = lambda lo, hi: (lo + (hi - lo) * rng.random((rows, d), dtype=F32)).astype(F32)
  st = {"table": u(-1, 1)}
  if kind in ("adagrad", "clippy", "ftrl"):
    st["accum"] = u(0.1, 1)
  if kind == "adam":
    st["m"], st["v"] = u(-0.1, 0.1), u(0.01, 0.5)
  if kind == "ftrl":
    st["linear"] = u(-0.1, 0.1)
  nz = list(neg_zero_rows)
  for k in ("table", "m", "v", "linear"):
    if k in st and nz:
      st[k][nz] = F32(-0.0)
  return st


def grads(rng, n, d):
  """Gradient rows of mixed exponents (2^-6 .. 2^6), so that any change of summation order shows in the bits."""
  u = rng.random((n, d), dtype=F32) * F32(2) - F32(1)
  return np.ldexp(u, rng.integers(-6, 7, size=(n, d)).astype(np.int32)).astype(F32)


def _cu(a):
  return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def run_gpu(ops, vname, dev, ids, g):
  """One step of the variant on the device tensors `dev` ({slot: tensor}), in place; returns {"factor": ...} for
  ClippyAdagrad.  `ids` and `g` are device tensors."""
  kind, kw = VARIANTS[vname]
  if kind == "sgd":
    ops.sparse_sgd_(dev["table"], ids, g, kw["lr"])
  elif kind == "adagrad":
    ops.sparse_adagrad_(dev["table"], dev["accum"], ids, g, kw["lr"], kw["eps"], kw["eps_inside_sqrt"])
  elif kind == "clippy":
    f = torch.full((), -1.0, device="cuda")
    ops.sparse_clippy_adagrad_(dev["table"], dev["accum"], ids, g, kw["lr"], kw["eps"], kw["var_rel"], kw["acc_rel"],
                               kw["abs_thr"], clip_accumulator_update=kw["clip"],
                               use_standard_accumulator_update=kw["standard"], clipping_factor=f)
    return {"factor": f}
  elif kind == "adam":
    ops.sparse_adam_(dev["table"], dev["m"], dev["v"], ids, g, float(ao.alpha(kw["lr"], kw["beta_1"], kw["beta_2"], kw["t"])),
                     kw["beta_1"], kw["beta_2"], kw["epsilon"], kw["lazy"])
  else:
    ops.sparse_ftrl_(dev["table"], dev["accum"], dev["linear"], ids, g, kw["lr"], kw["lr_power"], kw["l1"],
                     ops.ftrl_l2(kw["l2"], kw.get("beta", 0.0), kw["lr"]), kw.get("l2_shrinkage", 0.0))
  return {}


def _host(dev, extra):
  out = {k: t.cpu().numpy() for k, t in dev.items()}
  out.update({k: t.cpu().numpy() for k, t in extra.items()})
  return out


def fill_workspace(vname, n, d, rows, byte=0xA5):
  """Fills the cached scratch buffer the variant's next call will use with `byte`."""
  from recommenders_b200 import _ffi
  kind = VARIANTS[vname][0]
  lib = _ffi.lib()
  nbytes = {"sgd": lambda: lib.tfrs_sparse_sgd_workspace_bytes(n),
            "adagrad": lambda: lib.tfrs_sparse_adagrad_workspace_bytes(n, d),
            "clippy": lambda: lib.tfrs_sparse_clippy_adagrad_workspace_bytes(n, d),
            "adam": lambda: lib.tfrs_sparse_adam_workspace_bytes(n, rows),
            "ftrl": lambda: lib.tfrs_sparse_ftrl_workspace_bytes(n)}[kind]()
  _ffi.workspace(nbytes, torch.device("cuda", torch.cuda.current_device()), WS_SLOT[kind]).fill_(byte)


class Case:
  def __init__(self, name, rows, ids, g, neg_zero_rows=()):
    self.name, self.rows = name, rows
    self.ids = np.asarray(ids, np.int64)
    self.g = np.asarray(g, F32)
    self.d = self.g.shape[1]
    self.neg_zero_rows = tuple(neg_zero_rows)


def check_case(ops, case, variants=ALL, idts=IDTS, seed=0, scratch=False):
  """Runs every variant on the case (once per id dtype) and returns all mismatches as strings."""
  errs = []
  for idt in idts:
    if idt == torch.int32 and (case.ids.min(initial=0) < INT32_MIN or case.ids.max(initial=0) > INT32_MAX):
      continue
    ids_d, g_d = _cu(case.ids).to(idt), _cu(case.g)
    for vname in variants:
      st = init_states(vname, case.rows, case.d, seed, case.neg_zero_rows)
      want = reference(vname, st, case.ids, case.g)
      dev = {k: _cu(v) for k, v in st.items()}
      if scratch:
        fill_workspace(vname, case.ids.size, case.d, case.rows)
      got = _host(dev, run_gpu(ops, vname, dev, ids_d, g_d))
      errs += [f"[{case.name} {str(idt)[6:]}] {e}" for e in compare(vname, got, want, st, case.ids, case.g)]
  return errs


def _assert_clean(errs):
  assert not errs, f"{len(errs)} mismatches:\n" + "\n".join(errs[:40])


# ------------------------------------------------------------------------------------------------
# Case families
# ------------------------------------------------------------------------------------------------
def _place(rng, n, runs, fill_ids):
  """A batch of n ids: each (id, length) run's members at random positions, the other positions from `fill_ids` (in
  order).  Returns the ids."""
  members = np.concatenate([np.full(L, i, np.int64) for i, L in runs]) if runs else np.zeros(0, np.int64)
  assert members.size + len(fill_ids) == n, (members.size, len(fill_ids), n)
  ids = np.concatenate([members, np.asarray(fill_ids, np.int64)])
  return ids[rng.permutation(n)]


# 1. routes ----------------------------------------------------------------------------------------
ROUTE_NS = (1, 2, 3, 8191, 8192, 8193, 16383, 16384, 16385, 32768, 32769)


def route_case(n):
  """Duplicates and singletons (n >= 3), one run longer than AG_LONG from n = 200 up; d = 8 (float4 staging) for even n,
  d = 5 (scalar) for odd n."""
  rng = np.random.RandomState(n)
  d = 8 if n % 2 == 0 else 5
  rows = max(16, n)
  if n <= 3:
    ids = np.array([rows - 1, 3, rows - 1][:n] if n != 2 else [7, 7], np.int64)
  else:
    pool = rng.permutation(rows)
    ids = pool[:n].copy()
    hot = pool[:max(2, n // 50)]
    dup = rng.permutation(n)[:n // 3]
    ids[dup] = rng.choice(hot, size=dup.size)
    if n >= 200:
      ids[rng.permutation(n)[:70]] = hot[0]
  return Case(f"route_n{n}", rows, ids, grads(np.random.default_rng(n), n, d))


# 2. buckets ---------------------------------------------------------------------------------------
def one_bucket_case():
  """AG_RANK_MAX ids, every distinct id in the bucket of rows - 1, in runs of 1 to 100 members."""
  rows = 120_000
  rng = np.random.RandomState(21)
  cand = np.flatnonzero(ag_bucket(np.arange(rows)) == ag_bucket(rows - 1))
  lengths, k = [], 1
  while sum(lengths) < AG_RANK_MAX:
    lengths.append(min(k, AG_RANK_MAX - sum(lengths)))
    k = k % 100 + 1
  chosen = np.r_[rows - 1, rng.permutation(cand[cand != rows - 1])[:len(lengths) - 1]]
  ids = _place(rng, AG_RANK_MAX, list(zip(chosen, lengths)), [])
  return Case("one_bucket", rows, ids, grads(np.random.default_rng(21), AG_RANK_MAX, 4))


def bucket_sizes_case():
  """Eighteen buckets holding 0, 1, ..., 17 keys (a few distinct ids each), so that the AB_SPLIT slices of
  ceil(size / 8) keys come out empty, partial and full; every other bucket is empty."""
  rows = 50_000
  rng = np.random.RandomState(22)
  b_of = ag_bucket(np.arange(rows))
  ids = []
  for s in range(18):
    cand = np.flatnonzero(b_of == 10 + 7 * s)
    own = rng.permutation(cand)[:1 + s // 4]
    ids += list(own) + list(rng.choice(own, size=s - len(own))) if s >= len(own) else list(own[:s])
  ids = np.array(ids, np.int64)[rng.permutation(len(ids))]
  return Case("bucket_sizes", rows, ids, grads(np.random.default_rng(22), ids.size, 33))


def high_bits_case():
  """Ids next to id + 2^32 (same low 32 bits, out of range) and id + 2^33, with duplicates of the in-range ids."""
  rows = 5000
  rng = np.random.RandomState(23)
  base = rng.permutation(rows)[:300]
  ids = np.concatenate([base, base + 2 ** 32, base[:100], base[:50] + 2 ** 33, rng.randint(0, rows, size=500)])
  ids = ids[rng.permutation(ids.size)]
  return Case("high_bits", rows, ids, grads(np.random.default_rng(23), ids.size, 8))


# 3. run lengths x widths --------------------------------------------------------------------------
RUN_LENGTHS = (1, 2, 7, 8, 9, 31, 32, 33, 63, 64, 65, 66, 255, 256, 257, 258, 513)
WIDTHS = (1, 2, 3, 4, 5, 31, 32, 33, 64, 65, 100, 128, 129, 256, 257, 512, 513, 769, 1000, 1023, 1024)


def tile_runs(d):
  """T-1, T, T+1, 2T, 2T+1 (T = tile_rows(d)), and kT-1, kT, kT+1 for the first k with kT-1 > AG_LONG: runs that end one
  row before, at and after a tile edge inside the long-run kernel even where T itself is a warp-kernel length."""
  T = tile_rows(d)
  k = AG_LONG // T + 1
  while k * T - 1 <= AG_LONG:
    k += 1
  return {x for x in (T - 1, T, T + 1, 2 * T, 2 * T + 1, k * T - 1, k * T, k * T + 1) if x >= 1}


def run_lengths(d):
  return sorted(set(RUN_LENGTHS) | tile_runs(d))


def width_case(d, path, lengths=None, seed=None):
  """Every run length of run_lengths(d), each on its own id with its members scattered over the batch; a 257-member run
  on id 0 and the longest run on rows - 1, the largest id, which only out-of-range ids follow in (id, position) order;
  singletons; a few out-of-range ids.  "bucket": n <= AG_RANK_MAX.  "bitonic": singletons past AG_RANK_MAX."""
  lengths = run_lengths(d) if lengths is None else lengths
  rng = np.random.RandomState(d * 10 + (path == "bitonic") if seed is None else seed)
  members = sum(lengths) + 257
  oob = [-1, -1, -7, 0, 0]
  singles = 400 if path == "bucket" else AG_RANK_MAX + 101 - members - len(oob)
  rows = max(3000, members + singles + 10) if path == "bucket" else singles + len(lengths) + 200
  oob = [-1, rows, rows + 1, rows, INT32_MAX]
  pool = rng.permutation(np.arange(1, rows - 1))
  run_ids = [rows - 1 if L == max(lengths) else int(pool[i]) for i, L in enumerate(lengths)]
  runs = list(zip(run_ids, lengths)) + [(0, 257)]
  fill = list(pool[len(lengths):len(lengths) + singles]) + oob
  n = members + len(fill)
  ids = _place(rng, n, runs, fill)
  assert (path == "bucket") == (n <= AG_RANK_MAX)
  return Case(f"width_d{d}_{path}", rows, ids, grads(np.random.default_rng(d * 10 + 3), n, d))


# 4. many long runs --------------------------------------------------------------------------------
def many_long_case(d, path):
  """More long runs than the H100 has SMs: 200 runs of 65-80 members (bucket), 300 runs of 65 plus singletons (bitonic)."""
  rng = np.random.RandomState(40 + d)
  if path == "bucket":
    rows, lengths, singles = 1000, rng.randint(65, 81, size=200), 0
  else:
    rows, lengths, singles = 2000, np.full(300, 65), 800
  run_ids = rng.permutation(rows)[:len(lengths)]
  fill = rng.permutation(np.setdiff1d(np.arange(rows), run_ids))[:singles]
  n = int(lengths.sum()) + singles
  ids = _place(rng, n, list(zip(run_ids, lengths)), fill)
  return Case(f"many_long_d{d}_{path}", rows, ids, grads(np.random.default_rng(41 + d), n, d))


# 5. order of summation ----------------------------------------------------------------------------
BIG = F32(2.0 ** 24)
# summed in order: 2^24 + 1 rounds to 2^24 (a tie, to even) three times, -2^24 leaves 0, the last 1 gives 1.
# Reversed: 5.  Any pairing or tree of these terms gives something other than 1 as well.
PATTERN = np.array([BIG, 1, 1, 1, 1, -BIG, 1], F32)


def order_runs(d):
  """(name, member rows [L, d], neg_zero) for the order-of-summation family at width d."""
  T = tile_rows(d)
  scale = np.ldexp(F32(1), (np.arange(d) % 5 - 2)).astype(F32)        # per column: exact powers of two

  def pat(L, at):
    r = np.zeros((L, d), F32)
    r[at:at + len(PATTERN)] = PATTERN[:, None] * scale[None, :]
    return r

  def const(L, v):
    return np.full((L, d), v, F32)

  sub = np.ldexp(F32(1), -140).astype(F32)
  rng = np.random.default_rng(50 + d)
  inf_run = grads(rng, 70, d); inf_run[10] = np.inf; inf_run[40] = -np.inf
  nan_run = grads(rng, 120, d); nan_run[77] = np.nan
  sub_short = (np.arange(6 * d).reshape(6, d) % 7 - 3).astype(F32) * sub
  sub_long = (np.arange(90 * d).reshape(90, d) % 11 - 5).astype(F32) * sub
  pos_inf = grads(rng, 4, d); pos_inf[2] = np.inf
  neg_inf = grads(rng, 3, d); neg_inf[0] = -np.inf
  return [("in_one_step", pat(8, 0), False), ("across_steps", pat(20, 5), False), ("across_windows", pat(40, 29), False),
          ("long_in_tile", pat(300, 100), False), ("long_across_tile", pat(max(300, T + 40), T - 3), False),
          ("long_across_window", pat(300, AL_THREADS - 3), False),
          ("neg_zero_single", const(1, -0.0), True), ("neg_zero_short", const(5, -0.0), True),
          ("neg_zero_long", const(100, -0.0), True), ("subnormal_short", sub_short, False),
          ("subnormal_long", sub_long, False), ("pos_inf", pos_inf, False), ("neg_inf", neg_inf, False),
          ("inf_both_long", inf_run, False), ("nan_long", nan_run, False)]


def order_case(d, path):
  """The order_runs, each on its own id with members scattered, among singletons of ordinary gradients."""
  rng = np.random.RandomState(60 + d)
  runs = order_runs(d)
  members = sum(r.shape[0] for _, r, _ in runs)
  singles = 500 if path == "bucket" else AG_RANK_MAX + 50 - members
  rows = len(runs) + singles + 100
  pool = rng.permutation(rows)
  run_ids = pool[:len(runs)]
  fill = pool[len(runs):len(runs) + singles]
  n = members + singles
  perm = rng.permutation(n)
  ids = np.empty(n, np.int64)
  g = np.empty((n, d), F32)
  p = 0
  for rid, (_, r, _) in zip(run_ids, runs):
    slots = np.sort(perm[p:p + r.shape[0]])          # scattered, in the run's member order
    ids[slots] = rid
    g[slots] = r
    p += r.shape[0]
  ids[perm[p:]] = fill
  g[perm[p:]] = grads(np.random.default_rng(61 + d), singles, d)
  assert (path == "bucket") == (n <= AG_RANK_MAX)
  neg = [int(rid) for rid, (_, _, nz) in zip(run_ids, runs) if nz]
  return Case(f"order_d{d}_{path}", rows, ids, g, neg_zero_rows=neg)


# 6. ids -------------------------------------------------------------------------------------------
def id_edges(rows, idt):
  e = [-1, rows, rows + 1, INT32_MIN, INT32_MAX]
  if idt == torch.int64:
    e += [INT64_MIN, INT64_MAX, 2 ** 32, 2 ** 40 - 1, 2 ** 40, 2 ** 40 + 5, -2 ** 40]
  return e


def id_edge_case(idt):
  rows = 1000
  rng = np.random.RandomState(70)
  edges = id_edges(rows, idt)
  ids = rng.randint(0, rows, size=3000)
  ids[rng.permutation(3000)[:len(edges) * 20]] = np.repeat(edges, 20)
  ids[:4] = [0, rows - 1, 0, rows - 1]
  ids[rng.permutation(3000)[:70]] = rows - 1               # a long run on the largest id
  return Case(f"id_edges_{str(idt)[6:]}", rows, ids, grads(np.random.default_rng(70), 3000, 6))


# 7. position bits ---------------------------------------------------------------------------------
POSITION_VARIANTS = ("sgd", "adagrad_eps_inside", "ftrl_sqrt_shrink")


@functools.lru_cache(maxsize=1)
def position_case():
  """n = 2^24 - 1 at d = 1: runs of 1 to 8 members scattered over the whole batch, and one 300-member run whose members
  all sit at positions >= 2^23.  Returns (case, positions of the long run)."""
  n = MAX_N - 1
  rng = np.random.default_rng(7)
  long_pos = np.sort(rng.choice(np.arange(1 << 23, n), 300, replace=False))
  rest = n - 300
  counts = rng.integers(1, 9, size=rest // 4 + 1000)
  counts = counts[:np.searchsorted(np.cumsum(counts), rest) + 1]
  counts[-1] -= counts.sum() - rest
  short = np.repeat(np.arange(counts.size, dtype=np.int64), counts)
  rng.shuffle(short)
  ids = np.empty(n, np.int64)
  mask = np.ones(n, bool)
  mask[long_pos] = False
  ids[mask] = short
  ids[long_pos] = counts.size
  rows = counts.size + 1
  return Case("positions", rows, ids, grads(rng, n, 1)), long_pos


# ------------------------------------------------------------------------------------------------
# CPU: the case set stays on the code's edges; the references and their self-tests
# ------------------------------------------------------------------------------------------------
def _src(name):
  with open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "recommenders_b200", "csrc", name)) as f:
    return f.read()


def test_constants_and_shared_checks_match_the_sources():
  cu, cuh = _src("adagrad.cu"), _src("adagrad.cuh")
  src = cu + cuh
  for name, want in (("AG_RANK_MAX", AG_RANK_MAX), ("AG_TILE", AG_TILE), ("AB_BUCKETS", AB_BUCKETS), ("AB_SPLIT", AB_SPLIT),
                     ("AG_LONG", AG_LONG), ("AL_THREADS", AL_THREADS), ("AL_ROWS", AL_ROWS)):
    got = {int(v) for v in re.findall(rf"\b{name}\s*=\s*(\d+)\s*[,;]", src)}
    assert got == {want}, (name, got)
  budgets = re.findall(r"tile_rows = \((\d+) \* 1024\) / \(d \* 4\)", src)
  assert len(budgets) == 2 and {int(b) * 1024 for b in budgets} == {AL_SMEM}, budgets   # ag_apply_long and ag_run_sums
  # the bucket hash restated by ag_bucket()
  assert "(unsigned int)(key >> 24) ^ (unsigned int)(key >> 56)" in cu and "(id * 0x9E3779B1u) >> 24" in cu
  # the position field and n's limit
  assert "0xFFFFFFull" in cu and "0xFFFFFFull" in cuh and "<< 24" in cu
  # n's limit: ag_check_args holds it, and every sparse entry point calls ag_check_args under its own name
  # (tests/test_sparse_step_args.py also calls each entry point with n = 2^24)
  assert "n < (1ll << 24)" in cu
  for f in ("sgd.cu", "adagrad.cu", "clippy_adagrad.cu", "adam.cu", "ftrl.cu"):
    assert f'ag_check_args("sparse_{f[:-3]}", ' in _src(f), f


def test_run_lengths_cover_every_window_and_tile_edge():
  base = set(RUN_LENGTHS)
  for w in (32, 2 * 32):                                # the warp kernels' ballot windows up to AG_LONG
    assert {w - 1, w, w + 1} <= base, w
  assert {AG_LONG, AG_LONG + 1, AG_LONG + 2} <= base
  assert {AL_THREADS - 1, AL_THREADS, AL_THREADS + 1, AL_THREADS + 2, 2 * AL_THREADS + 1} <= base   # long-kernel windows
  assert {1, 7, 8, 9} <= base                          # 8 rows in flight per warp step
  for d in WIDTHS:
    T = tile_rows(d)
    L = set(run_lengths(d))
    assert {T - 1, T, T + 1} - {0} <= L, d
    long_edges = {x % T for x in L if x > AG_LONG}
    assert {0, 1, T - 1} <= long_edges, (d, T)          # long runs ending at, one past and one before a tile edge
  assert {T for T in map(tile_rows, WIDTHS)} >= {256, 163, 127, 64, 63, 32, 31, 21, 16}
  assert {d for d in WIDTHS if d > 2 * AL_THREADS} and max(WIDTHS) == 4 * AL_THREADS    # columns u = 0..3 per thread


@pytest.mark.parametrize("path", ["bucket", "bitonic"])
def test_width_cases_are_what_they_say(path):
  for d in (1, 100, 1024):
    c = width_case(d, path)
    inr = (c.ids >= 0) & (c.ids < c.rows)
    vals, cnt = np.unique(c.ids[inr], return_counts=True)
    runs = dict(zip(vals.tolist(), cnt.tolist()))
    assert sorted(k for k in cnt if k > 1) == sorted([k for k in run_lengths(d) if k > 1] + [257]), d
    assert runs[0] == 257 and runs[c.rows - 1] == max(run_lengths(d)) and vals.max() == c.rows - 1
    assert (~inr).sum() >= 5
    assert (c.ids.size <= AG_RANK_MAX) == (path == "bucket")
    first = np.flatnonzero(c.ids == c.rows - 1)
    assert np.diff(first).max() > 1                   # members scattered


def test_route_and_long_run_cases_straddle_the_boundaries():
  ns = set(ROUTE_NS)
  assert {AG_RANK_MAX - 1, AG_RANK_MAX, AG_RANK_MAX + 1} <= ns
  assert {AG_TILE - 1, AG_TILE, AG_TILE + 1} <= ns
  assert {4 * AG_TILE, 4 * AG_TILE + 1} <= ns and padded(4 * AG_TILE + 1) == 2 * padded(4 * AG_TILE)
  assert {1, 2, 3} <= ns
  for n in ROUTE_NS:
    c = route_case(n)
    assert c.ids.size == n
    if n >= 3:
      _, cnt = np.unique(c.ids, return_counts=True)
      assert (cnt == 1).any() and (cnt > 1).any(), n
    if n >= 200:
      assert cnt.max() > AG_LONG, n
  for d in (64, 1000):
    for path in ("bucket", "bitonic"):
      c = many_long_case(d, path)
      _, cnt = np.unique(c.ids, return_counts=True)
      assert (cnt > AG_LONG).sum() > H100_SMS and (c.ids.size <= AG_RANK_MAX) == (path == "bucket")


def test_bucket_cases_collide_under_the_restated_hash():
  c = one_bucket_case()
  assert c.ids.size == AG_RANK_MAX
  vals, cnt = np.unique(c.ids, return_counts=True)
  assert len(set(ag_bucket(vals).tolist())) == 1 and vals.max() == c.rows - 1
  assert set(cnt.tolist()) == set(range(1, 101))
  c = bucket_sizes_case()
  sizes = np.bincount(ag_bucket(c.ids).astype(np.int64), minlength=AB_BUCKETS)
  assert set(sizes.tolist()) == set(range(18)) and (sizes > 0).sum() == 17
  per = -(-sizes // AB_SPLIT)
  filled = [np.clip(sizes - per * s, 0, per) for s in range(AB_SPLIT)]
  assert any(((f == 0) & (sizes > 0)).any() for f in filled)                  # an empty slice of a non-empty bucket
  assert any(((f > 0) & (f < per)).any() for f in filled)                     # a partial slice
  c = high_bits_case()
  inr = c.ids[c.ids < c.rows]
  hi = c.ids[c.ids >= c.rows]
  assert np.isin(hi & 0xFFFFFFFF, inr).all() and (hi >> 32 >= 1).all()
  assert ((hi >> 32) == 1).any() and ((hi >> 32) == 2).any()


def test_sgd_reference_matches_the_loop_oracle():
  rng = np.random.RandomState(80)
  rows, d, n = 60, 7, 900
  ids = rng.randint(-3, rows + 3, size=n)
  ids[rng.permutation(n)[:100]] = 5
  g = grads(np.random.default_rng(80), n, d)
  t = init_states("sgd", rows, d, 80)["table"]
  assert np.array_equal(_bits(_sgd_ref(t, ids, g, 0.3)), _bits(ebo.sgd_sparse(t, ids, g, 0.3)))


def test_adagrad_reference_matches_the_c_oracle():
  rng = np.random.RandomState(81)
  rows, d, n = 500, 9, 5000
  ids = rng.randint(-3, rows + 3, size=n)
  ids[rng.permutation(n)[:300]] = 17
  for case in (Case("random", rows, ids, grads(np.random.default_rng(81), n, d)), order_case(3, "bucket")):
    for inside in (True, False):
      st = init_states("adagrad_eps_inside", case.rows, case.d, 81, case.neg_zero_rows)
      want = orc.sparse_adagrad(st["table"], st["accum"], case.ids, case.g, 0.1, 1e-3, inside)
      got = _adagrad_ref(st["table"], st["accum"], case.ids, case.g, 0.1, 1e-3, inside)
      for a, b in zip(got, want):
        assert not _mismatch(a, b).any(), (case.name, inside)


# where summing from +0.0f shows: a -0.0 sum changes the sign of a zero update (SGD does not sum, FTRL's rule maps a
# -0.0 and a +0.0 gradient to the same bits)
ZERO_START_SHOWS = ("adagrad_eps_inside", "adagrad_eps_outside", "clippy_flags0", "clippy_flags2", "adam", "adam_lazy")


def test_order_cases_reject_other_summation_orders():
  """The reference result of the order family differs from the same step with each run's sum started from +0.0f (where
  that can show) and with each run's members reversed (for SGD, the occurrences applied last to first), under the same
  comparison the GPU tests use: a kernel that summed either way would fail them."""
  case = order_case(3, "bucket")
  assert sorted(set(RUN_LENGTHS) & {8, 20, 40}) == [8]
  heads, s = run_sums(case.ids, case.g, case.rows)
  p = {name: i for i, (name, _, _) in enumerate(order_runs(3))}
  assert len(p) == 15
  for vname in ALL:
    st = init_states(vname, case.rows, case.d, 0, case.neg_zero_rows)
    want = reference(vname, st, case.ids, case.g)
    if VARIANTS[vname][0] == "sgd":
      ids_r, g_r = case.ids[::-1].copy(), case.g[::-1].copy()
      assert compare(vname, reference(vname, st, ids_r, g_r), want, st, case.ids, case.g), vname
      continue
    for mode in ("zero_start", "reversed"):
      h, sm = run_sums(case.ids, case.g, case.rows, mode)
      errs = compare(vname, reference(vname, st, h, sm), want, st, case.ids, case.g)
      assert bool(errs) == (mode == "reversed" or vname in ZERO_START_SHOWS), (vname, mode, errs)
    # and the in-order sum over the run heads alone is the reference itself
    assert not compare(vname, reference(vname, st, heads, s), want, st, case.ids, case.g), vname


def test_pattern_sums():
  with np.errstate(all="ignore"):
    acc = PATTERN[0]
    for x in PATTERN[1:]:
      acc = F32(acc + x)
    rev = PATTERN[-1]
    for x in PATTERN[-2::-1]:
      rev = F32(rev + x)
  assert acc == 1 and rev == 5
  c = order_case(64, "bucket")
  heads, s = run_sums(c.ids, c.g, c.rows)
  _, z = run_sums(c.ids, c.g, c.rows, "zero_start")
  _, r = run_sums(c.ids, c.g, c.rows, "reversed")
  assert (_bits(s) != _bits(z)).any() and (_mismatch(s, r)).any()


# ------------------------------------------------------------------------------------------------
# GPU: 1. routes
# ------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("n", ROUTE_NS)
def test_routes(ops, n):
  _assert_clean(check_case(ops, route_case(n)))


# 2. buckets
@gpu
@pytest.mark.parametrize("which", ["one_bucket", "bucket_sizes", "high_bits"])
def test_buckets(ops, which):
  case = {"one_bucket": one_bucket_case, "bucket_sizes": bucket_sizes_case, "high_bits": high_bits_case}[which]()
  _assert_clean(check_case(ops, case, idts=(torch.int64,) if which == "high_bits" else IDTS))


# 3. run lengths x widths
@gpu
@pytest.mark.parametrize("path", ["bucket", "bitonic"])
@pytest.mark.parametrize("d", WIDTHS)
def test_run_lengths_at_width(ops, d, path):
  _assert_clean(check_case(ops, width_case(d, path), idts=(torch.int32,) if d % 2 else (torch.int64,)))


@gpu
def test_sgd_wide_rows_and_one_long_run(ops):
  """SGD has no width limit: d = 1500 with every run length, and one run of 20000 members among singletons."""
  errs = check_case(ops, width_case(1500, "bucket", lengths=list(RUN_LENGTHS), seed=15), variants=("sgd",))
  rng = np.random.RandomState(16)
  rows, n = 3000, 20_400
  ids = _place(rng, n, [(rows - 1, 20_000)], list(rng.permutation(rows - 1)[:400]))
  errs += check_case(ops, Case("sgd_run_20000", rows, ids, grads(np.random.default_rng(16), n, 1500)), variants=("sgd",))
  _assert_clean(errs)


# 4. many long runs
@gpu
@pytest.mark.parametrize("path", ["bucket", "bitonic"])
@pytest.mark.parametrize("d", [64, 1000])
def test_more_long_runs_than_sms(ops, d, path):
  _assert_clean(check_case(ops, many_long_case(d, path), idts=(torch.int32,)))


# 5. order of summation
@gpu
@pytest.mark.parametrize("path", ["bucket", "bitonic"])
@pytest.mark.parametrize("d", [3, 64])
def test_order_of_summation(ops, d, path):
  _assert_clean(check_case(ops, order_case(d, path), idts=(torch.int64,)))


# 6. ids
@gpu
@pytest.mark.parametrize("idt", IDTS)
def test_id_edge_values(ops, idt):
  _assert_clean(check_case(ops, id_edge_case(idt), idts=(idt,)))


@gpu
@pytest.mark.parametrize("idt", IDTS)
def test_only_out_of_range_ids(ops, idt):
  """No row changes, except that Adam (not lazy) decays every row; ClippyAdagrad's factor is exactly 1."""
  rows, d = 300, 5
  edges = id_edges(rows, idt)
  ids = np.array(edges * 10, np.int64)
  case = Case("only_out_of_range", rows, ids, grads(np.random.default_rng(90), ids.size, d))
  errs = check_case(ops, case, idts=(idt,))
  ids_d, g_d = _cu(ids).to(idt), _cu(case.g)
  for vname in ALL:
    st = init_states(vname, rows, d, 1)
    dev = {k: _cu(v) for k, v in st.items()}
    got = _host(dev, run_gpu(ops, vname, dev, ids_d, g_d))
    if vname == "adam":
      assert (_bits(got["m"]) != _bits(st["m"])).all(axis=1).all() and (_bits(got["table"]) != _bits(st["table"])).any(1).all()
    else:
      for k in st:
        assert np.array_equal(_bits(got[k]), _bits(st[k])), (vname, k)
    if "factor" in got:
      assert _bits(got["factor"]) == _bits(F32(1)), vname
  _assert_clean(errs)


# 7. position bits
@gpu
@pytest.mark.parametrize("vname", POSITION_VARIANTS)
def test_positions_past_2_to_the_23(ops, vname):
  """Every position bit of the key: members at positions >= 2^23 on the bitonic path, short runs and a long run.  The
  reference sums the long run on its own (the rows are disjoint, so the two steps compose)."""
  case, long_pos = position_case()
  st = init_states(vname, case.rows, 1, 3)
  short = case.ids.copy()
  short[long_pos] = -1
  want = reference(vname, reference(vname, st, short, case.g), case.ids[long_pos], case.g[long_pos])
  dev = {k: _cu(v) for k, v in st.items()}
  got = _host(dev, run_gpu(ops, vname, dev, _cu(case.ids).to(torch.int32), _cu(case.g)))
  _assert_clean(compare(vname, got, want))


@gpu
@pytest.mark.parametrize("kind", ["sgd", "adagrad", "clippy", "adam", "ftrl"])
def test_n_of_2_to_the_24_is_refused(ops, kind):
  vname = {"sgd": "sgd", "adagrad": "adagrad_eps_inside", "clippy": "clippy_flags0", "adam": "adam",
           "ftrl": "ftrl_sqrt_shrink"}[kind]
  st = init_states(vname, 8, 1, 4)
  dev = {k: _cu(v) for k, v in st.items()}
  ids = torch.zeros(MAX_N, dtype=torch.int32, device="cuda")
  g = torch.ones((MAX_N, 1), device="cuda")
  with pytest.raises(ValueError, match=r"2\^24"):
    run_gpu(ops, vname, dev, ids, g)
  for k in st:
    assert np.array_equal(_bits(dev[k].cpu().numpy()), _bits(st[k])), (kind, k)


# 8. alignment
def align_case(d):
  rng = np.random.RandomState(100 + d)
  rows = 500
  run_ids = rng.permutation(rows)[:5]
  fill = list(rng.permutation(np.setdiff1d(np.arange(rows), run_ids))[:200]) + [-1, rows]
  runs = list(zip(run_ids, (300, 70, 65, 20, 3)))
  n = 458 + len(fill)
  return Case(f"align_d{d}", rows, _place(rng, n, runs, fill), grads(np.random.default_rng(100 + d), n, d))


def _offset_copy(x, floats):
  """A contiguous copy of x that starts `floats` floats into its storage."""
  buf = torch.empty(x.numel() + 4, device="cuda")
  v = buf[floats:floats + x.numel()].view(x.shape)
  v.copy_(x)
  assert v.data_ptr() % 16 == 4 * floats and v.is_contiguous()
  return v


@gpu
@pytest.mark.parametrize("d", [4, 64, 1024])
def test_misaligned_grad_rows(ops, d):
  """grad_rows starting 4, 8 and 12 bytes into its storage take the scalar staging and give the aligned call's bits."""
  case = align_case(d)
  ids_d, g_d = _cu(case.ids), _cu(case.g)
  errs = []
  for vname in ALL:
    st = init_states(vname, case.rows, d, 5)
    dev = {k: _cu(v) for k, v in st.items()}
    aligned = _host(dev, run_gpu(ops, vname, dev, ids_d, g_d))
    errs += compare(vname, aligned, reference(vname, st, case.ids, case.g), st, case.ids, case.g)
    for off in (1, 2, 3):
      dev = {k: _cu(v) for k, v in st.items()}
      got = _host(dev, run_gpu(ops, vname, dev, ids_d, _offset_copy(g_d, off)))
      errs += [f"offset {4 * off} B: {e}" for e in compare(vname, got, aligned)]
      errs += [f"offset {4 * off} B, exact bits: {k}" for k in got if not np.array_equal(_bits(got[k]), _bits(aligned[k]))]
  _assert_clean(errs)


@gpu
@pytest.mark.parametrize("slot", ["table", "m", "v"])
@pytest.mark.parametrize("d", [4, 64, 1024])
def test_misaligned_adam_slots(ops, d, slot):
  """Adam's table, m or v starting 4, 8 or 12 bytes into its storage: the decay pass takes single columns and every
  array gets the aligned call's bits."""
  case = align_case(d)
  ids_d, g_d = _cu(case.ids), _cu(case.g)
  errs = []
  for vname in ("adam", "adam_lazy"):
    st = init_states(vname, case.rows, d, 6)
    dev = {k: _cu(v) for k, v in st.items()}
    aligned = _host(dev, run_gpu(ops, vname, dev, ids_d, g_d))
    errs += compare(vname, aligned, reference(vname, st, case.ids, case.g))
    for off in (1, 2, 3):
      dev = {k: _cu(v) for k, v in st.items()}
      dev[slot] = _offset_copy(dev[slot], off)
      got = _host(dev, run_gpu(ops, vname, dev, ids_d, g_d))
      errs += [f"{slot} at offset {4 * off} B: {vname}.{k}" for k in got if not np.array_equal(_bits(got[k]), _bits(aligned[k]))]
  _assert_clean(errs)


# 9. scratch
@gpu
@pytest.mark.parametrize("path", ["bucket", "bitonic"])
def test_garbage_scratch_and_repeatability(ops, path):
  """The cached workspace filled with 0xA5 bytes before each call changes nothing, and two identical calls give
  identical bits."""
  case = width_case(64, path, lengths=[1, 2, 9, 33, 65, 257, 300], seed=9)
  errs = check_case(ops, case, idts=(torch.int64,), seed=11, scratch=True)
  ids_d, g_d = _cu(case.ids), _cu(case.g)
  for vname in ALL:
    st = init_states(vname, case.rows, case.d, 11)
    outs = []
    for _ in range(2):
      dev = {k: _cu(v) for k, v in st.items()}
      fill_workspace(vname, case.ids.size, case.d, case.rows)
      outs.append(_host(dev, run_gpu(ops, vname, dev, ids_d, g_d)))
    errs += [f"{vname}.{k}: two calls differ" for k in outs[0] if not np.array_equal(_bits(outs[0][k]), _bits(outs[1][k]))]
  _assert_clean(errs)


# 10. TreeAH grouping
@gpu
@pytest.mark.parametrize("n", [1, 2, 8191, 8192, 8193, 16384, 16385, 100000])
def test_tree_ah_group(ops, n):
  """order = positions by (leaf, position) over the in-range leaves, then the out-of-range positions in order; offsets =
  the first sorted slot of each leaf.  Every third leaf is empty; the workspace starts as 0xA5 garbage."""
  from recommenders_b200 import _ffi
  rng = np.random.RandomState(n)
  L = max(4, n // 20)
  leaf = rng.choice(np.flatnonzero(np.arange(L) % 3 != 1), size=n).astype(np.int64)
  oob = np.array([-1, L, L + 5, 2 ** 40, 2 ** 40 - 1, INT64_MIN, INT64_MAX], np.int64)
  if n >= 100:
    k = rng.permutation(n)[:n // 50]
    leaf[k] = rng.choice(oob, size=k.size)
  elif n == 2:
    leaf[:] = [L + 5, 0]
  _ffi.workspace(_ffi.lib().tfrs_tree_ah_group_workspace_bytes(n), torch.device("cuda", torch.cuda.current_device()),
                 "tree_ah").fill_(0xA5)
  order, offsets = ops.tree_ah_group(_cu(leaf), L)
  order, offsets = order.cpu().numpy(), offsets.cpu().numpy()
  inr = (leaf >= 0) & (leaf < L)
  pos = np.flatnonzero(inr)
  want = np.r_[pos[np.argsort(leaf[pos], kind="stable")], np.flatnonzero(~inr)]
  assert np.array_equal(order, want)
  assert np.array_equal(offsets, np.searchsorted(np.sort(leaf[inr]), np.arange(L + 1), side="left"))
