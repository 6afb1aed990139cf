"""CPU checks of tests/test_gpu_exact_anchor_edges.py: the constants of the exact SGEMM (csrc/sgemm.cuh), its batch
split-K, the row select (csrc/rowselect.cuh), the exact scan's chunk plan and the list merges (csrc/topk.cu) and the
exact Dense (csrc/dense.cu) are read back from the sources, and the GPU file's case lists must still hit every edge they
define.  A changed constant then fails here instead of silently dropping coverage.  Also a NumPy self-test of the
split-K and bias-gradient references: they must tell the kernels' summation orders from near misses."""
import importlib.util
import os
import re

import numpy as np
import pytest

from oracle import oracle as orc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "recommenders_b200", "csrc")


def _src(name):
  with open(os.path.join(CSRC, name)) as f:
    return f.read()


def _int(pattern, text):
  m = re.search(pattern, text)
  assert m, pattern
  return int(m.group(1))


@pytest.fixture(scope="module")
def gpu():
  path = os.path.join(ROOT, "tests", "test_gpu_exact_anchor_edges.py")
  spec = importlib.util.spec_from_file_location("_exact_anchor_edges", path)
  mod = importlib.util.module_from_spec(spec)
  spec.loader.exec_module(mod)
  return mod


@pytest.fixture(scope="module")
def C():
  sg, topk, rs, dense = _src("sgemm.cuh"), _src("topk.cu"), _src("rowselect.cuh"), _src("dense.cu")
  c = {
      "SG_BM": _int(r"SG_BM = (\d+)", sg), "SG_BN": _int(r"SG_BN = (\d+)", sg), "SG_BK": _int(r"SG_BK = (\d+)", sg),
      "SKINNY": _int(r"const bool skinny = N <= (\d+);", sg),
      "SPLIT_ROWS": _int(r"sgemm_batch_splits\(long long B\) \{ long long z = ceil_div\(B, (\d+)\)", sg),
      "SPLIT_MAX": _int(r"z > (\d+) \? \d+ : z", sg),
      "CAP_MIN": _int(r"return c < (\d+) \? \d+ : c; \}", rs),
      "CAP_MUL": _int(r"int c = pow2_ceil\((\d+) \* k\);", rs),
      "ROOM_DIV": _int(r"const int min_room = cap / (\d+);", rs),
      "SCAN_MB": _int(r"budget : \(size_t\)(\d+) << 20", topk),
      "SCAN_MIN_NC": _int(r"if \(nc < (\d+)\) nc = \d+;", topk),
      "SCAN_ALIGN": _int(r"/ \(\(size_t\)Q \* 4\)\) / (\d+) \* \d+;", topk),
      "SHRINK_MIN": _int(r"ws_bytes > fixed \+ \(size_t\)Q \* (\d+) \* 4", topk),
      "MS_MAX_LISTS": _int(r"constexpr int MS_MAX_LISTS = (\d+);", topk),
      "MS_SMEM_KB": _int(r"region \* 24 > (\d+) \* 1024", topk),
      "SCAN_MAX_K": _int(r"k > 0 && k <= (\d+), \"topk_scan", topk),
      "DENSE_NARROW_N": _int(r"constexpr int DENSE_NARROW_N = (\d+);", dense),
      "DENSE_COL_SPLITS": _int(r"constexpr int DENSE_COL_SPLITS = (\d+);", dense),
      "CROSS_COL_SPLITS": _int(r"constexpr int CROSS_COL_SPLITS = (\d+);", _src("cross.cu")),
  }
  # the shapes of the formulas the GPU file restates
  assert "const int kps = (int)(ceil_div(ceil_div(K, splits), SG_BK) * SG_BK);" in sg
  assert "if (pos < total && cap - cnt >= min_room) continue;" in rs
  assert "keep = cnt < k ? cnt : k;" in rs
  return c


def cap_of(C, k):
  c = 1
  while c < C["CAP_MUL"] * k:
    c <<= 1
  return max(c, C["CAP_MIN"])


def test_sgemm_cases_hit_every_tile_slab_and_loader_edge(gpu, C):
  BM, BN, BK, SK = C["SG_BM"], C["SG_BN"], C["SG_BK"], C["SKINNY"]
  assert {1, BM - 1, BM, BM + 1, 2 * BM + 1} <= set(gpu.SG_M)
  assert {1, SK - 1, SK, SK + 1, BN - 1, BN, BN + 1} <= set(gpu.SG_N)
  Ks = set(gpu.SG_K)
  assert {0, 1, BK - 1, BK, BK + 1, 2 * BK - 1, 2 * BK + 1} <= Ks
  assert {k % 4 for k in Ks if k > BK} == {0, 1, 2, 3} and {k % 4 for k in Ks if 0 < k < BK} == {0, 1, 2, 3}
  assert any(k > 4 * BK and k % BK for k in Ks)           # several full slabs, then a partial one
  assert set(gpu.SG_MODES) == {(a, b) for a in (False, True) for b in (False, True)}
  cases = gpu.SG_CASES
  for axis, values in ((0, gpu.SG_M), (1, gpu.SG_N), (2, gpu.SG_K)):
    assert {c[axis] for c in cases} == set(values)
  # loader fallbacks: every misaligned base, an ld that breaks float4 and one that keeps it with a row gap
  assert set(gpu.SG_OFFSETS) == {1, 2, 3} and set(gpu.SG_LD_PAD) == {1, 4}
  assert any(K % 4 == 0 for _, _, K in gpu.SG_LD_SHAPES) and any(K % BK for _, _, K in gpu.SG_LD_SHAPES)
  assert all(K % BK for K in gpu.SG_NEG_ZERO_K) and {K % 4 for K in gpu.SG_NEG_ZERO_K} >= {1, 3}
  assert any(K > BK for K in gpu.SG_NEG_ZERO_K) and any(K < BK for K in gpu.SG_NEG_ZERO_K)


def test_split_k_cases_hit_every_range_edge(gpu, C):
  R, Z = C["SPLIT_ROWS"], C["SPLIT_MAX"]
  Bs = set(gpu.SPLIT_B)
  assert {R, R + 1, 2 * R + 1, Z * R, Z * R + 1} <= Bs
  assert any(B > Z * R and B % (Z * R) and B % 16 for B in Bs)     # at the cap, ragged last range
  n_ranges = {len(gpu.sgemm_batch_ranges(B)) for B in Bs}
  assert {1, 2, 3, Z} <= n_ranges and max(n_ranges) == Z
  for B in Bs:                                                    # the restated ranges tile [0, B) in order
    r = gpu.sgemm_batch_ranges(B)
    assert r[0][0] == 0 and r[-1][1] == B and all(a[1] == b[0] for a, b in zip(r, r[1:]))
    want = min(max(-(-B // R), 1), Z)
    if want > 1:
      kps = -(-(-(-B // want)) // C["SG_BK"]) * C["SG_BK"]
      assert all(hi - lo == kps for lo, hi in r[:-1])
  K, N = gpu.DENSE_BWD_KN
  assert K < 64 or N < 64                                         # dense_tc needs K >= 64 and N >= 64
  assert gpu.CROSS_BWD_D < 64
  assert gpu.cdiv(70000, C["DENSE_COL_SPLITS"]) == gpu.cdiv(70000, 64) and C["CROSS_COL_SPLITS"] == 64
  Ns = {n for _, _, n in gpu.DENSE_FWD_CASES}
  assert {C["DENSE_NARROW_N"], C["DENSE_NARROW_N"] + 1, C["SKINNY"], C["SKINNY"] + 1, C["SG_BN"], C["SG_BN"] + 1} <= Ns
  assert all(b < 1024 or k < 64 or n < 64 for b, k, n in gpu.DENSE_FWD_CASES)


def test_row_select_cases_hit_every_cap_tier(gpu, C):
  ks = gpu.SEL_K
  assert max(ks) == C["SCAN_MAX_K"] and 1 in ks and 2 in ks
  assert all(gpu.rowselect_cap(k) == cap_of(C, k) for k in range(1, C["SCAN_MAX_K"] + 1))
  tiers = sorted({cap_of(C, k) for k in range(1, C["SCAN_MAX_K"] + 1)})
  for cap in tiers:                 # both sides of every tier switch, each tier's first and last k
    lo = min(k for k in range(1, C["SCAN_MAX_K"] + 1) if cap_of(C, k) == cap)
    hi = max(k for k in range(1, C["SCAN_MAX_K"] + 1) if cap_of(C, k) == cap)
    assert {lo, hi} <= set(ks) or (lo == 1 and hi in ks)
    if hi > 1:
      assert hi - 1 in ks or hi - 1 == lo
  for k in ks:
    cap = cap_of(C, k)
    n = gpu.sel_counts(k)
    assert {c for c in (k - 1, k, k + 1, cap - 1, cap, cap + 1) if c > 0} <= set(n)
    assert max(n) > 4 * cap                                            # several compactions
  assert set(gpu.SEL_PATTERNS) >= {"equal", "inf", "zeros"}


def test_compaction_boundary_cases(gpu, C):
  """The boundary test puts k + m = 3 cap / 4 + delta in the buffer after the first compaction; min_room = cap / 4
  must separate delta = 0 (keep filling) from delta = 1 (compact)."""
  for k in gpu.SEL_K:
    cap = cap_of(C, k)
    room = cap // C["ROOM_DIV"]
    for delta in (-1, 0, 1):
      cnt = 3 * cap // 4 + delta
      assert (cap - cnt >= room) == (delta <= 0)


def test_scan_plan_cases(gpu, C):
  Q, N, k = gpu.CHUNK_QNK
  nc = (C["SCAN_MB"] << 20) // (Q * 4) // C["SCAN_ALIGN"] * C["SCAN_ALIGN"]
  nc = min(max(nc, C["SCAN_MIN_NC"]), -(-N // 128) * 128)
  assert nc == gpu.scan_nc(Q, N)
  assert nc >= C["SCAN_MIN_NC"] and nc % C["SCAN_ALIGN"] == 0 and N > 2 * nc and N % nc
  for Q, N, k, extra in gpu.SHRINK_CASES:
    fixed = 2 * gpu.state_bytes(Q, k)
    ws = fixed + extra
    assert ws > fixed + Q * C["SHRINK_MIN"] * 4                      # the shrink branch is taken
    budget = ws - fixed - 256
    nc = max(budget // (Q * 4) // 128 * 128, C["SCAN_MIN_NC"])
    assert (Q * nc * 4 + 255) // 256 * 256 + fixed <= ws             # and the shrunk plan fits
    assert nc < N and N % nc                                         # several chunks, a ragged last one
  assert any(k > C["SCAN_MAX_K"] // 2 for _, _, k, _ in gpu.SHRINK_CASES)


def _region(n_lists, k_in, k_out):
  tot = n_lists * k_in
  ko = min(k_out, tot)
  region, n, c = tot, n_lists, k_in
  while n > 2:
    n = (n + 1) // 2
    c = min(2 * c, ko)
    region = max(region, n * c)
  return region


def test_merge_cases_hit_the_tree_merge_limits(gpu, C):
  limit = C["MS_SMEM_KB"] * 1024
  cases = gpu.TREE_MERGE_CASES
  ns = {n for n, _, _ in cases}
  assert {C["MS_MAX_LISTS"], C["MS_MAX_LISTS"] + 1} <= ns
  under = [_region(n, ki, ko) * 24 for n, ki, ko in cases if n <= C["MS_MAX_LISTS"] and _region(n, ki, ko) * 24 <= limit]
  over = [_region(n, ki, ko) * 24 for n, ki, ko in cases if _region(n, ki, ko) * 24 > limit]
  assert any(limit - 24 < r <= limit for r in under) and any(limit < r <= limit + 48 for r in over)
  assert any(n > 2 and limit - 96 < _region(n, ki, ko) * 24 <= limit for n, ki, ko in cases)
  assert all(ko <= C["SCAN_MAX_K"] for _, _, ko in cases + gpu.SORT_MERGE_CASES)
  for n, ki, ko in gpu.SORT_MERGE_CASES:
    assert n * ki > cap_of(C, ko)
  assert max(ko for _, _, ko in gpu.SORT_MERGE_CASES) == C["SCAN_MAX_K"]
  assert cap_of(C, gpu.OVERRIDE_K) > cap_of(C, gpu.OVERRIDE_K - 1)


def test_tc_unaligned_cases():
  path = os.path.join(ROOT, "tests", "test_gpu_exact_anchor_edges.py")
  src = open(path).read()
  ds = [int(x) for x in re.search(r"TC_UNALIGNED_D = \[([\d, ]+)\]", src).group(1).split(",")]
  assert any(d % 32 == 0 and d != 64 for d in ds) and any(d % 4 == 0 and d % 32 for d in ds) and 64 in ds
  tc = _src("topk_tc.cu")
  assert "(d & 31) == 0" in tc and "(d & 3) == 0" in tc and "p.d == 64" in tc


# ---- the references reject near misses
def test_split_k_reference_rejects_reversed_partials(gpu):
  rng = np.random.RandomState(0)
  B = 70000
  x = rng.normal(size=(B, 3)).astype(np.float32); g = rng.normal(size=(B, 5)).astype(np.float32)
  ref, rev = gpu.split_k_ref(x, g), gpu.split_k_ref(x, g, reverse=True)
  assert len(gpu.sgemm_batch_ranges(B)) == 16
  assert not np.array_equal(ref.view(np.uint32), rev.view(np.uint32))
  np.testing.assert_allclose(ref, x.astype(np.float64).T @ g.astype(np.float64), rtol=1e-4, atol=1e-3)


def test_db_reference_rejects_pairwise_sum(gpu):
  B = 4097
  dz = np.stack([gpu.adversarial_column(B), np.random.RandomState(1).normal(size=B).astype(np.float32)], 1)
  ref = gpu.dense_db_ref(dz)
  pairwise = np.float32(np.sum(np.ascontiguousarray(dz[:, 0], np.float64)))   # a contiguous 1-D sum is pairwise
  assert ref[0] != pairwise


def test_chain_reference_rejects_a_zero_padded_tail():
  t = np.float32(2.0 ** -80)
  for K in (1, 3, 17, 33):
    a = np.full((2, K), -t, np.float32); b = np.full((3, K), t, np.float32)
    exact = orc.scores(a, b)
    padded = orc.scores(np.pad(a, ((0, 0), (0, 16 - K % 16))), np.pad(b, ((0, 0), (0, 16 - K % 16))))
    assert (exact.view(np.uint32) == 0x80000000).all()
    assert (padded.view(np.uint32) == 0).all()
