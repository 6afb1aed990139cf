"""Edge cases of the embedding gather (csrc/gather.cu, K1) and of DotInteraction (csrc/dot_interaction.cu): every gather
route and the per-batch route choice past 32 tables, every warp-chunk lane count, hot-row staging on both sides of its
rule at every row width, id edge values, the empty batch, and DotInteraction at its feature and shared-memory limits.

Gather reference: NumPy `table[ids]` with a zero row for an id outside [0, rows), compared bit for bit.  Tables hold
arbitrary bit patterns (NaN payloads, signed zeros, subnormals), so a kernel that did arithmetic on the values instead of
copying them would show.  Every output starts filled with SENTINEL, and the columns no table writes must keep it.

The host's choices, restated here (`route`, `staging`):
  route, per batch of 32 tables: "chunk" (gather_warpchunk_kernel) when `out`, every table, every column offset and
    `out_ld` are 16-byte aligned and every width is 4 L floats with L a power of two <= 32; "vec" (gather_kernel<VEC>)
    when only the power-of-two rule fails; "scalar" (gather_kernel<!VEC>) otherwise.
  staging, per 512-row CTA of the chunk kernel: H = min(16 KB / row bytes, rows); thread t of the CTA holds ids t and
    t + 256; the CTA stages table[0:H] in shared memory when the number of THREADS holding an id in [0, H) exceeds H / 2.

DotInteraction: the forward is the oracle's fmaf chain, compared bit for bit.  The backward is compared per element with
the float64 oracle under the bar of `_di_backward_bar` (derivation there; DESIGN section 2).
The GPU tests are marked one by one; the case-set checks and the bar self-test run without a GPU.
"""
import re

import numpy as np
import pytest
import torch

from oracle import oracle as orc

gpu = pytest.mark.gpu

SENTINEL = -7.0
SENTINEL_BITS = int(np.array(SENTINEL, np.float32).view(np.int32))
INT32_MIN, INT32_MAX = -2 ** 31, 2 ** 31 - 1
INT64_MIN, INT64_MAX = -2 ** 63, 2 ** 63 - 1

# csrc/gather.cu
GT_MAX_TABLES = 32
GT_THREADS = 256
GT_CTA_CHUNKS = 2
GT_CTA_ROWS = GT_THREADS * GT_CTA_CHUNKS
GT_HOT_BYTES = 16384
# csrc/dot_interaction.cu
DI_WARPS = 4
DI_MAX_F = 64
DI_SMEM = 200 * 1024

IDTS = (torch.int32, torch.int64)
NS = (1, 31, 33, 511, 513, 4099)           # one row, partial warps on both sides of 32, partial CTAs on both sides of 512
WIDTHS = {1: "scalar", 3: "scalar", 4: "chunk", 8: "chunk", 12: "vec", 16: "chunk", 20: "vec", 32: "chunk", 48: "vec",
          64: "chunk", 96: "vec", 128: "chunk", 132: "vec"}
HOT_WIDTHS = (4, 8, 16, 32, 64, 128)
DI_MODES = ((False, False), (True, False), (False, True), (True, True))   # (self_interaction, skip_gather)


@pytest.fixture(scope="module")
def ops():
  from recommenders_b200 import ops as o
  return o


# ------------------------------------------------------------------------------------------------
# The host's route rule and the chunk kernel's staging rule, restated
# ------------------------------------------------------------------------------------------------
def route(dims, col_offsets, out_ld, aligned):
  """The kernel tfrs_gather_f32 launches for one batch of at most 32 tables.  `aligned`: `out` and every table start on
  a 16-byte boundary."""
  vec = aligned and out_ld % 4 == 0 and all(d % 4 == 0 for d in dims) and all(c % 4 == 0 for c in col_offsets)
  if not vec:
    return "scalar"
  lanes = [d // 4 for d in dims]
  return "chunk" if all(1 <= L <= 32 and L & (L - 1) == 0 for L in lanes) else "vec"


def routes(dims, col_offsets, out_ld, aligned):
  """One route per batch of GT_MAX_TABLES tables, in launch order."""
  return [route(dims[t:t + GT_MAX_TABLES], col_offsets[t:t + GT_MAX_TABLES], out_ld, aligned)
          for t in range(0, len(dims), GT_MAX_TABLES)]


def hot_capacity(width):
  """Rows of `width` floats the 16 KB staging buffer holds: 1024 >> log2(width / 4)."""
  return GT_HOT_BYTES // (4 * width)


def staging(ids, rows, width):
  """The chunk kernel's decision for each CTA: (staged [CTAs], threads holding a hot id [CTAs], H).  A thread counts once
  however many of its two ids are hot.  A CTA has 256 threads, so it can stage only when H / 2 < 256: for widths 4 and 8
  (H = 1024 and 512 rows of a large table) that takes a table of fewer than 512 rows, which is then staged whole.  A change
  to GT_HOT_BYTES or GT_CTA_CHUNKS that moves these limits makes test_hot_row_cases_cover_both_sides_of_the_rule fail."""
  ids = np.asarray(ids, np.int64)
  H = min(hot_capacity(width), rows)
  ctas = -(-len(ids) // GT_CTA_ROWS)
  pad = np.full(ctas * GT_CTA_ROWS, -1, np.int64)
  pad[:len(ids)] = ids
  hot = (pad >= 0) & (pad < H)
  n_hot = hot.reshape(ctas, GT_CTA_CHUNKS, GT_THREADS).any(axis=1).sum(axis=1)  # CTA row ch * 256 + t belongs to thread t
  return (n_hot > H // 2) & (H > 0), n_hot, H


# ------------------------------------------------------------------------------------------------
# Gather cases: tables of arbitrary bits, ids, and the bit-exact reference with sentinel columns
# ------------------------------------------------------------------------------------------------
def _table(rng, rows, width):
  return rng.randint(INT32_MIN, INT32_MAX + 1, size=(rows, width), dtype=np.int64).astype(np.int32).view(np.float32)


def _expected(tables, ids, col_offsets, n, cols):
  """int32 bits of the output: each table's rows (zero for an out-of-range id) in its columns, SENTINEL elsewhere."""
  exp = np.full((n, cols), SENTINEL_BITS, np.int32)
  for tab, idx, off in zip(tables, ids, col_offsets):
    tb = np.ascontiguousarray(tab).view(np.int32)
    idx = np.asarray(idx, np.int64)
    ok = (idx >= 0) & (idx < tb.shape[0])
    rows = np.zeros((n, tb.shape[1]), np.int32)
    rows[ok] = tb[idx[ok]]
    exp[:, off:off + tb.shape[1]] = rows
  return exp


def _bits(t):
  return t.detach().contiguous().view(torch.int32).cpu().numpy()


def _gather_check(ops, tables, ids, idt, col_offsets, cols, pad_left=0, out_ld=None, dev_tables=None):
  """ops.gather into columns [pad_left, pad_left + cols) of a SENTINEL-filled buffer of `out_ld` columns; checks the
  whole buffer bit for bit.  Returns the route the host rule predicts for each batch of tables."""
  n = len(ids[0])
  out_ld = cols if out_ld is None else out_ld
  buf = torch.full((n, out_ld), SENTINEL, device="cuda")
  out = buf[:, pad_left:pad_left + cols]
  dev_tables = [torch.from_numpy(t).cuda() for t in tables] if dev_tables is None else dev_tables
  dev_ids = [torch.from_numpy(np.asarray(i, np.int64)).to(device="cuda", dtype=idt) for i in ids]
  got = ops.gather(dev_tables, dev_ids, out=out, col_offsets=col_offsets)
  assert got.data_ptr() == out.data_ptr()
  exp = _expected(tables, ids, [pad_left + c for c in col_offsets], n, out_ld)
  g = _bits(buf)
  if not np.array_equal(g, exp):
    r, c = np.argwhere(g != exp)[0]
    raise AssertionError(f"{int((g != exp).sum())} words differ; first [{r}, {c}]: got {g[r, c]:#010x} want {exp[r, c]:#010x}")
  aligned = out.data_ptr() % 16 == 0 and all(t.data_ptr() % 16 == 0 for t in dev_tables)
  return routes([int(t.shape[1]) for t in dev_tables], list(col_offsets), out_ld, aligned)


def _width_case(width, n, seed):
  """Two tables of one width side by side (3000 rows, and 50 rows so that ids repeat), 4 sentinel columns after them;
  ids run past both ends of each table."""
  rng = np.random.RandomState(seed)
  tables = [_table(rng, 3000, width), _table(rng, 50, width)]
  ids = [rng.randint(-3, 3003, size=n), rng.randint(-2, 53, size=n)]
  return tables, ids, [0, width], 2 * width + 4


CHUNK_WIDTHS = (4, 128, 8, 64, 16, 32)


def _many_tables_case(order, n=700, seed=40):
  """40 tables: batch 0 is tables 0..31, batch 1 tables 32..39.  "chunk_then_vec": batch 0 mixes every chunk width
  (4 and 128 together), batch 1 has widths of 3, 5, 12 and 24 lanes.  "vec_then_chunk": one 12-float table turns batch 0
  to VEC, batch 1 is all chunk widths."""
  rng = np.random.RandomState(seed)
  widths = [CHUNK_WIDTHS[t % len(CHUNK_WIDTHS)] for t in range(32)]
  if order == "chunk_then_vec":
    widths += [48, 12, 20, 96, 48, 12, 20, 96]
  else:
    widths[17] = 12
    widths += [CHUNK_WIDTHS[t % len(CHUNK_WIDTHS)] for t in range(8)]
  rows = [100 + 37 * t for t in range(40)]
  tables = [_table(rng, r, w) for r, w in zip(rows, widths)]
  ids = [rng.randint(-2, r + 2, size=n) for r in rows]
  offs = list(np.cumsum([0] + widths[:-1]))
  return tables, ids, [int(o) for o in offs], int(sum(widths)) + 8


# ------------------------------------------------------------------------------------------------
# Hot-row cases: for each width, tables below and above the staging capacity, skewed ids, and CTAs built to sit one
# thread on each side of the rule
# ------------------------------------------------------------------------------------------------
def _boundary_cta(rng, H, n_hot_threads, hot_id, cold_id):
  """512 ids of one CTA in which exactly `n_hot_threads` threads hold a hot id.  Hot threads hold (hot, hot), (hot, cold)
  or (cold, hot) in turn, so the CTA has more hot ids than hot threads."""
  first, second = np.empty(GT_THREADS, np.int64), np.empty(GT_THREADS, np.int64)
  hot_threads = set(rng.permutation(GT_THREADS)[:n_hot_threads].tolist())
  k = 0
  for t in range(GT_THREADS):
    if t in hot_threads:
      first[t], second[t] = ((hot_id(), hot_id()), (hot_id(), cold_id()), (cold_id(), hot_id()))[k % 3]
      k += 1
    else:
      first[t], second[t] = cold_id(), cold_id()
  return np.concatenate([first, second])   # CTA row t is thread t's first id, row 256 + t its second


def hot_cases(width):
  """[(name, rows, ids)] for one width.  Every case ends in a partial CTA whose last warp is partial (77 rows)."""
  rng = np.random.RandomState(1000 + width)
  cap = hot_capacity(width)
  tail = 77
  cases = []

  # the whole table fits the buffer (H = rows; fewer than 512 rows, so widths 4 and 8 can stage): CTA 0 uniform, CTA 1
  # nearly all ids out of range, CTA 2 uniform; the partial last CTA has too few threads to stage unless H is tiny
  small = min(cap - 1, 300)
  oob = lambda: int(rng.choice([-1, small, small + 1]))
  ids = rng.randint(0, small, size=3 * GT_CTA_ROWS + tail)
  ids[GT_CTA_ROWS:2 * GT_CTA_ROWS] = [oob() for _ in range(GT_CTA_ROWS)]
  ids[GT_CTA_ROWS + 5:GT_CTA_ROWS + 15] = rng.randint(0, small, size=10)
  cases.append(("whole_table", small, ids))

  # the same table, one CTA with small // 2 hot threads (not staged) and one with small // 2 + 1 (staged); only ids
  # outside the table are cold here
  hot = lambda: int(rng.randint(0, small))
  ids = np.concatenate([_boundary_cta(rng, small, small // 2, hot, oob), _boundary_cta(rng, small, small // 2 + 1, hot, oob),
                        rng.randint(-1, small + 2, size=tail)])
  cases.append(("whole_table_boundary", small, ids))

  # a table larger than the buffer with a hot prefix: CTA 0 has 5 hot ids, CTAs 1.. draw rows * u^k, k rising, so the
  # hot share rises from CTA to CTA; every CTA also has ids above H and a few out of range
  rows = 4 * cap + 3
  parts = [np.concatenate([rng.randint(0, cap, size=5), rng.randint(cap, rows, size=GT_CTA_ROWS - 5)])]
  for k in (1, 3, 8, 24, 64):
    parts.append(np.floor(rows * rng.uniform(size=GT_CTA_ROWS) ** k).astype(np.int64))
  parts.append(np.floor(rows * rng.uniform(size=tail) ** 8).astype(np.int64))
  ids = np.concatenate(parts)
  for c in range(6):
    ids[c * GT_CTA_ROWS + 7] = cap + 1 + c       # at least one id above H in every full CTA
    ids[c * GT_CTA_ROWS + 300] = rows + c         # out of range
    ids[c * GT_CTA_ROWS + 301] = -1 - c
  cases.append(("skewed", rows, ids))

  # the large table with CTAs one thread on each side of H / 2 (H = cap); cold ids are table rows at or above H
  cold = lambda: int(rng.randint(cap, rows))
  hot = lambda: int(rng.randint(0, cap))
  if cap // 2 + 1 <= GT_THREADS:
    ids = np.concatenate([_boundary_cta(rng, cap, cap // 2, hot, cold), _boundary_cta(rng, cap, cap // 2 + 1, hot, cold),
                          [-1, rows], rng.randint(0, rows, size=tail - 2)])
    cases.append(("prefix_boundary", rows, ids))
  return cases


def test_gather_case_set_covers_every_route():
  """The route rule sends each parametrized case where its name says, and the cases reach every route: chunk at each L in
  1..32, VEC at lane counts that are not powers of two, scalar for odd widths and for each misaligned layout."""
  seen = set()
  for w, want in WIDTHS.items():
    tables, ids, offs, cols = _width_case(w, 1, 0)
    assert route([w, w], offs, cols, True) == want, w
    seen.add((want, w // 4 if want != "scalar" else None))
  assert {L for r, L in seen if r == "chunk"} == {1, 2, 4, 8, 16, 32}
  assert {L for r, L in seen if r == "vec"} >= {3, 5, 12, 24, 33}
  assert ("scalar", None) in seen
  assert route([32, 32], [0, 32], 68, True) == "chunk"
  for name, (dims, offs, out_ld, aligned) in _layout_cases().items():
    assert route(dims, offs, out_ld, aligned) == "scalar", name
  for order, want in (("chunk_then_vec", ["chunk", "vec"]), ("vec_then_chunk", ["vec", "chunk"])):
    tables, ids, offs, cols = _many_tables_case(order)
    assert routes([t.shape[1] for t in tables], offs, cols, True) == want
  assert {4, 128} <= {t.shape[1] for t in _many_tables_case("chunk_then_vec")[0][:32]}


def _layout_cases():
  """Layouts that force the scalar kernel at width 32: (dims, col_offsets, out_ld, aligned) as the host sees them."""
  return {"out_column_view": ([32, 32], [0, 32], 68, False),     # `out` starts one float into its buffer
          "out_ld_odd": ([32, 32], [0, 32], 67, True),
          "col_offset_odd": ([32, 32], [0, 34], 68, True),
          "table_view": ([32, 32], [0, 32], 64, False)}          # a table starts 4 bytes into its storage


def test_hot_row_cases_cover_both_sides_of_the_rule():
  for w in HOT_WIDTHS:
    cap = hot_capacity(w)
    by_name = {name: (rows, ids, *staging(ids, rows, w)) for name, rows, ids in hot_cases(w)}
    for name, (rows, ids, staged, n_hot, H) in by_name.items():
      assert len(ids) % GT_CTA_ROWS and len(ids) % 32, name          # a partial last CTA and a partial last warp
      assert ids.min() < 0 and ids.max() >= rows, name               # ids outside the table on both sides
    # the table smaller than the buffer is staged whole, in some CTAs and not in others, at every width
    rows, ids, staged, n_hot, H = by_name["whole_table"]
    assert rows < cap and rows < 512 and H == rows
    assert staged.any() and not staged.all(), w
    rows, ids, staged, n_hot, H = by_name["whole_table_boundary"]
    assert list(n_hot[:2]) == [H // 2, H // 2 + 1] and list(staged[:2]) == [False, True], w
    assert ((ids[:GT_CTA_ROWS] >= 0) & (ids[:GT_CTA_ROWS] < H)).sum() > H // 2   # a count of ids would have staged CTA 0
    # the table larger than the buffer: every full skewed CTA has ids below and above H
    rows, ids, staged, n_hot, H = by_name["skewed"]
    assert H == cap < rows
    full = ids[:len(ids) // GT_CTA_ROWS * GT_CTA_ROWS].reshape(-1, GT_CTA_ROWS)
    assert (((full >= 0) & (full < H)).any(1) & (full >= H).any(1)).all(), w
    if w <= 8:
      # H / 2 >= 256 threads: a CTA of a large table can never stage at widths 4 and 8
      assert H // 2 >= GT_THREADS and not staged.any(), w
      assert "prefix_boundary" not in by_name
    else:
      assert staged.any() and not staged.all(), w
      rows, ids, staged, n_hot, H = by_name["prefix_boundary"]
      assert H == cap and list(n_hot[:2]) == [H // 2, H // 2 + 1] and list(staged[:2]) == [False, True], w
      assert ((ids[:GT_CTA_ROWS] >= 0) & (ids[:GT_CTA_ROWS] < H)).sum() > H // 2


# ------------------------------------------------------------------------------------------------
# 1. Gather routes and shapes
# ------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("idt", IDTS)
@pytest.mark.parametrize("width", list(WIDTHS))
def test_gather_route_per_width(ops, width, idt):
  for n in NS:
    tables, ids, offs, cols = _width_case(width, n, seed=width * 7919 + n)
    assert _gather_check(ops, tables, ids, idt, offs, cols) == [WIDTHS[width]], (width, n)


@gpu
@pytest.mark.parametrize("idt", IDTS)
@pytest.mark.parametrize("layout", list(_layout_cases()))
def test_gather_routes_forced_by_layout(ops, layout, idt):
  """Width 32 would take the chunk kernel; each layout makes one alignment condition fail."""
  rng = np.random.RandomState(5)
  for n in (33, 513, 4099):
    tables = [_table(rng, 900, 32), _table(rng, 40, 32)]
    ids = [rng.randint(-1, 901, size=n), rng.randint(0, 41, size=n)]
    if layout == "out_column_view":
      r = _gather_check(ops, tables, ids, idt, [0, 32], 64, pad_left=1, out_ld=68)
    elif layout == "out_ld_odd":
      r = _gather_check(ops, tables, ids, idt, [0, 32], 64, out_ld=67)
    elif layout == "col_offset_odd":
      r = _gather_check(ops, tables, ids, idt, [0, 34], 68)       # columns 32 and 33 stay SENTINEL
    else:
      store = torch.from_numpy(np.concatenate([_table(rng, 1, 1).reshape(-1), tables[0].reshape(-1)])).cuda()
      view = store[1:].view(900, 32)
      assert view.data_ptr() % 16 == 4
      r = _gather_check(ops, tables, ids, idt, [0, 32], 64, dev_tables=[view, torch.from_numpy(tables[1]).cuda()])
    assert r == ["scalar"], (layout, n, r)


@gpu
@pytest.mark.parametrize("idt", IDTS)
@pytest.mark.parametrize("order", ["chunk_then_vec", "vec_then_chunk"])
def test_gather_more_than_32_tables(ops, order, idt):
  tables, ids, offs, cols = _many_tables_case(order)
  want = ["chunk", "vec"] if order == "chunk_then_vec" else ["vec", "chunk"]
  assert _gather_check(ops, tables, ids, idt, offs, cols) == want


@gpu
@pytest.mark.parametrize("idt", IDTS)
@pytest.mark.parametrize("width", [3, 12, 32])
def test_gather_id_edge_values(ops, width, idt):
  """Ids just outside the table, the id type's extremes and 2^40, all in one batch, on each route; then a one-row table
  (H = 1: a CTA stages as soon as one thread holds id 0)."""
  rng = np.random.RandomState(width)
  rows = 1000
  edges = [-1, rows, rows + 1, INT32_MIN, INT32_MAX, 0, rows - 1]
  if idt == torch.int64:
    edges += [2 ** 40, -2 ** 40, INT64_MIN, INT64_MAX, 2 ** 32, 2 ** 32 + 5]
  ids = rng.randint(0, rows, size=1100)
  ids[rng.permutation(1100)[:len(edges) * 20]] = np.repeat(edges, 20)
  ids[:len(edges)] = edges
  tables = [_table(rng, rows, width)]
  assert _gather_check(ops, tables, [ids], idt, [0], width + 4) == [WIDTHS[width]]
  one = [_table(rng, 1, width)]
  for n in (1, 40, 1100):
    ids1 = rng.choice(np.array([0, 0, 0, 1, -1, 2] + ([2 ** 40] if idt == torch.int64 else [INT32_MAX]), np.int64), size=n)
    _gather_check(ops, one, [ids1], idt, [0], width + 4)


@gpu
@pytest.mark.parametrize("idt", IDTS)
def test_gather_empty_batch(ops, idt):
  """n = 0 returns an empty [0, width] result, as tf.gather does (an empty CUDA tensor's pointer is NULL)."""
  tables = [torch.randn((10, 32), device="cuda"), torch.randn((7, 5), device="cuda")]
  ids = [torch.empty((0,), dtype=idt, device="cuda") for _ in tables]
  out = ops.gather(tables, ids)
  assert tuple(out.shape) == (0, 37) and out.dtype == torch.float32 and out.is_cuda
  out = ops.gather(tables, ids, out=torch.empty((0, 40), device="cuda"), col_offsets=[8, 0])
  assert tuple(out.shape) == (0, 40)
  import recommenders_b200 as tfrs
  emb = tfrs.layers.embedding.Embedding(10, 16)
  assert tuple(emb(torch.empty((0,), dtype=idt, device="cuda")).shape) == (0, 16)


@gpu
def test_gather_deterministic_and_independent_of_output_contents(ops):
  """Two calls give the same bits, and so does a call into an output full of garbage (NaNs, infinities, anything), on
  every route and with CTAs that stage hot rows."""
  rng = np.random.RandomState(77)
  n = 3 * GT_CTA_ROWS + 45
  for widths in ([32, 128, 4], [48, 20], [3, 32]):
    tables = [torch.from_numpy(_table(rng, 600, w)).cuda() for w in widths]
    ids = [torch.from_numpy(np.floor(600 * rng.uniform(size=n) ** 8).astype(np.int64) - 1).cuda() for _ in widths]
    first = _bits(ops.gather(tables, ids))
    assert np.array_equal(_bits(ops.gather(tables, ids)), first)
    garbage = torch.from_numpy(_table(rng, n, sum(widths))).cuda()
    assert np.array_equal(_bits(ops.gather(tables, ids, out=garbage)), first)


@gpu
def test_gather_route_rule_matches_the_kernels_launched(ops):
  """The kernels the host launches (read from torch.profiler) are the ones `route` predicts, in order, with the id type
  as the kernel's template argument."""
  from torch.profiler import ProfilerActivity, profile
  rng = np.random.RandomState(3)
  calls = []
  for idt in IDTS:
    for w in WIDTHS:
      tables, ids, offs, cols = _width_case(w, 513, seed=w)
      calls.append((idt, tables, ids, offs, cols, {}))
    for order in ("chunk_then_vec", "vec_then_chunk"):
      calls.append((idt, *_many_tables_case(order), {}))
    tables = [_table(rng, 300, 32), _table(rng, 30, 32)]
    ids = [rng.randint(0, 300, size=600), rng.randint(0, 30, size=600)]
    calls.append((idt, tables, ids, [0, 32], 64, dict(pad_left=1, out_ld=68)))
    calls.append((idt, tables, ids, [0, 32], 64, dict(out_ld=67)))
    calls.append((idt, tables, ids, [0, 34], 68, {}))
  torch.cuda.synchronize()
  want = []
  with profile(activities=[ProfilerActivity.CUDA]) as prof:
    for idt, tables, ids, offs, cols, kw in calls:
      want += [(r, "int" if idt == torch.int32 else "long") for r in _gather_check(ops, tables, ids, idt, offs, cols, **kw)]
    torch.cuda.synchronize()
  got = []
  for e in sorted(prof.events(), key=lambda e: e.time_range.start):
    m = re.search(r"gather_(warpchunk_kernel<(\w+)>|kernel<(\w+), (true|false|\(bool\)[01])>)", e.name)
    if m:
      r = "chunk" if m.group(2) else ("vec" if m.group(4) in ("true", "(bool)1") else "scalar")
      got.append((r, m.group(2) or m.group(3)))
  assert got == want


# ------------------------------------------------------------------------------------------------
# 2. Hot-row staging at every lane count
# ------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("idt", IDTS)
@pytest.mark.parametrize("width", HOT_WIDTHS)
def test_gather_hot_rows(ops, width, idt):
  """Every case of `hot_cases` (staged and unstaged CTAs side by side, see test_hot_row_cases_cover_both_sides_of_the_rule)
  into columns [4, 4 + width) of an output with sentinel columns on both sides."""
  rng = np.random.RandomState(width)
  for name, rows, ids in hot_cases(width):
    table = _table(rng, rows, width)
    assert _gather_check(ops, [table], [ids], idt, [4], width + 8) == ["chunk"], name


# ------------------------------------------------------------------------------------------------
# 3. DotInteraction at its limits
# ------------------------------------------------------------------------------------------------
def _di_feats(rng, B, F, d):
  return rng.normal(size=(B, F, d)).astype(np.float32)


def _di_oracle(feats, self_interaction, skip_gather):
  return orc.dot_interaction([feats[:, f] for f in range(feats.shape[1])], self_interaction, skip_gather)


def _kept(F, self_interaction):
  i, j = np.meshgrid(np.arange(F), np.arange(F), indexing="ij")
  return (j <= i) if self_interaction else (j < i)


def _sym_grad(g, F, self_interaction, skip_gather):
  """G' [B, F, F] float64: the upstream gradient at the kept (i, j) entries, symmetrised (the diagonal counts twice)."""
  g = np.asarray(g, np.float64)
  kept = _kept(F, self_interaction)
  if skip_gather:
    G = np.where(kept[None], g.reshape(-1, F, F), 0.0)
  else:
    G = np.zeros((g.shape[0], F, F))
    G[:, kept] = g
  return G + G.transpose(0, 2, 1)


def _gamma(n, u):
  return n * u / (1.0 - n * u)


def _di_backward_bar(feats, g, self_interaction, skip_gather):
  """Per-element bar of dE [B, F, d].

  The kernel computes dE_ik = fl(... fmaf(c_i1, e_1k, fmaf(c_i0, e_0k, +0))), j = 0..F-1 ascending, with c_ij = G'_ij
  read from the fp32 upstream gradient (2·g_ii on the diagonal, an exact doubling).  Each fmaf rounds once: s_j =
  (s_{j-1} + c_ij e_jk)(1 + δ_j), |δ_j| <= u = 2^-24.  Term j is multiplied by at most F factors (1 + δ), so
  |got - exact| <= γ_F Σ_j |c_ij| |e_jk|, γ_F = F u / (1 - F u) (Higham, Accuracy and Stability, §3.1).  The float64
  oracle reads the same fp32 features and gradient, so no input rounding enters; its own summation error is at most
  γ_F(2^-53) of the same sum, added.  Where a partial sum is subnormal a step errs by up to 2^-150 absolute instead:
  F·2^-149 covers that with the growth of later steps."""
  F = feats.shape[1]
  S = np.abs(_sym_grad(g, F, self_interaction, skip_gather)) @ np.abs(feats.astype(np.float64))
  return (_gamma(F, 2.0 ** -24) + _gamma(F, 2.0 ** -53)) * S + F * 2.0 ** -149


def _di_backward_check(got, ref, bar, what):
  err = np.abs(np.asarray(got, np.float64) - ref)
  bad = ~(err <= bar)
  if bad.any():
    i = tuple(np.argwhere(bad)[0])
    raise AssertionError(f"{what}: {int(bad.sum())} elements miss the bar; first {i}: got {got[i]!r} ref {ref[i]!r} "
                         f"err {err[i]:.3e} bar {bar[i]:.3e}")


def _fmaf_chain_backward(feats, g, self_interaction, skip_gather):
  """The kernel's arithmetic on the CPU: dE[b] = C[b] . E[b] as fmaf chains over j ascending (the oracle's C scores())."""
  B, F, d = feats.shape
  C = _sym_grad(g, F, self_interaction, skip_gather).astype(np.float32)   # exact: fp32 values, doubled on the diagonal
  return np.stack([orc.scores(C[b], np.ascontiguousarray(feats[b].T)) for b in range(B)])


@pytest.mark.parametrize("mode", DI_MODES)
def test_dot_interaction_backward_bar_rejects_a_doubled_term(mode):
  """CPU self-test of `_di_backward_bar`: the kernel's fmaf chain, run on the CPU, is inside the bar; the same chain with
  one feature's contribution counted twice, or with the diagonal counted once, is not."""
  si, sg = mode
  rng = np.random.RandomState(11)
  B, F, d = 3, 33, 17
  feats = _di_feats(rng, B, F, d)
  g = rng.normal(size=(B, F * F if sg else (F * (F + 1) // 2 if si else F * (F - 1) // 2))).astype(np.float32)
  ref = orc.dot_interaction_grads([feats[:, f] for f in range(F)], g, si, sg)
  bar = _di_backward_bar(feats, g, si, sg)
  chain = _fmaf_chain_backward(feats, g, si, sg)
  _di_backward_check(chain, ref, bar, "fmaf chain")
  Gs = _sym_grad(g, F, si, sg)
  j0 = 7
  doubled = chain + Gs[:, :, j0, None] * feats[:, None, j0, :].astype(np.float64)
  assert (np.abs(doubled - ref) > bar).mean() > 0.9
  if si:
    diag_once = chain - 0.5 * np.einsum("bii,bik->bik", Gs, feats.astype(np.float64))
    assert (np.abs(diag_once - ref) > bar).mean() > 0.9


def _di_forward_shapes():
  """(F, d, B) for the forward grid: every F x d at B in {1, 3, 5}; B = 4097 where the oracle stays cheap."""
  out = []
  for F in (1, 2, 33, 63, 64):
    for d in (1, 31, 33, 135):
      out.append((F, d, (1, 3, 5, 4097) if F * F * d <= 64 * 64 * 33 else (1, 3, 5)))
  return out


@gpu
@pytest.mark.parametrize("F,d,Bs", _di_forward_shapes())
def test_dot_interaction_forward_bit_exact(ops, F, d, Bs):
  """F = 64 with d = 135 fills the 200 KB staging limit of the backward exactly; B not a multiple of DI_WARPS = 4 leaves
  the last CTA's warps partly idle.  Packed-triangle positions up to F(F+1)/2 - 1 = 2079 go through the sqrtf guess."""
  rng = np.random.RandomState(F * 1000 + d)
  assert DI_WARPS * (F * (d + 1) + F * F) * 4 <= DI_SMEM
  for B in Bs:
    feats = _di_feats(rng, B, F, d)
    x = torch.from_numpy(feats).cuda()
    for si, sg in DI_MODES:
      exp = _di_oracle(feats, si, sg)
      got = ops.dot_interaction(x, si, sg)
      assert tuple(got.shape) == exp.shape, (B, si, sg)
      assert np.array_equal(_bits(got), exp.view(np.int32)), (B, si, sg)


@gpu
def test_dot_interaction_outside_the_staging_limits_raises(ops):
  """F = 64, d = 136 needs 201 KB of staging and F = 65 exceeds DI_MAX_F: both raise NotImplementedError, from the op
  and from the layer.  (The reference layer takes any F.)"""
  import recommenders_b200 as tfrs
  layer = tfrs.layers.feature_interaction.DotInteraction
  assert DI_WARPS * (64 * 137 + 64 * 64) * 4 > DI_SMEM
  for F, d in ((64, 136), (DI_MAX_F + 1, 8)):
    x = torch.randn((3, F, d), device="cuda")
    for si, sg in DI_MODES:
      with pytest.raises(NotImplementedError):
        ops.dot_interaction(x, si, sg)
      with pytest.raises(NotImplementedError):
        layer(self_interaction=si, skip_gather=sg)([x[:, f] for f in range(F)])


@gpu
def test_dot_interaction_empty_batch(ops):
  """B = 0: an empty [0, out_dim] result and an empty gradient, in every mode (an empty CUDA tensor's pointer is NULL)."""
  for si, sg in DI_MODES:
    x = torch.empty((0, 5, 8), device="cuda").requires_grad_(True)
    out = ops.dot_interaction(x, si, sg)
    assert tuple(out.shape) == (0, ops.lib().tfrs_dot_interaction_out_dim(5, int(si), int(sg)))
    out.backward(torch.empty_like(out))
    assert tuple(x.grad.shape) == (0, 5, 8)


DI_BACKWARD_SHAPES = ((1, 31, 5), (2, 1, 3), (2, 135, 4097), (33, 33, 4097), (63, 31, 5), (64, 135, 1), (64, 135, 5),
                      (64, 1, 4097))


@gpu
@pytest.mark.parametrize("F,d,B", DI_BACKWARD_SHAPES)
def test_dot_interaction_backward_per_element(ops, F, d, B):
  """Every element of dE within `_di_backward_bar` of the float64 oracle, in all four modes.  F = 1 without
  self-interaction has no outputs: its gradient is exactly zero."""
  rng = np.random.RandomState(F * 7 + d * 13 + B)
  feats = _di_feats(rng, B, F, d)
  for si, sg in DI_MODES:
    od = ops.lib().tfrs_dot_interaction_out_dim(F, int(si), int(sg))
    g = rng.normal(size=(B, od)).astype(np.float32)
    x = torch.from_numpy(feats).cuda().requires_grad_(True)
    ops.dot_interaction(x, si, sg).backward(torch.from_numpy(g).cuda())
    got = x.grad.cpu().numpy()
    ref = orc.dot_interaction_grads([feats[:, f] for f in range(F)], g, si, sg)
    _di_backward_check(got, ref, _di_backward_bar(feats, g, si, sg), f"F={F} d={d} B={B} self={si} skip={sg}")
    if od == 0:
      assert not got.any()


@gpu
@pytest.mark.parametrize("F,d,B", [(64, 135, 5), (33, 31, 4097), (2, 8, 3)])
@pytest.mark.parametrize("self_interaction", [False, True])
def test_dot_interaction_skip_gather_ignores_masked_gradient(ops, F, d, B, self_interaction):
  """With skip_gather the upstream gradient is [B, F*F]; entries above the diagonal (and on it without self-interaction)
  are not outputs of the layer.  Filled with 1e30 they must give the same bits as zeros.  (NaN would test nothing: TF
  would turn NaN * 0 into NaN.)"""
  rng = np.random.RandomState(F + d + B)
  feats = torch.from_numpy(_di_feats(rng, B, F, d)).cuda()
  kept = _kept(F, self_interaction).reshape(-1)
  g = rng.normal(size=(B, F * F)).astype(np.float32)
  grads = []
  for fill in (0.0, 1e30):
    x = feats.clone().requires_grad_(True)
    ops.dot_interaction(x, self_interaction, True).backward(torch.from_numpy(np.where(kept, g, np.float32(fill))).cuda())
    grads.append(_bits(x.grad))
  assert np.array_equal(grads[0], grads[1])


@gpu
@pytest.mark.parametrize("F,d,B", [(33, 32, 5), (64, 135, 3), (8, 7, 4097)])
def test_dot_interaction_mixed_data_exact(ops, F, d, B):
  """Integer features (every dot exact), e_1 = -e_0, all-(-0.0) and all-(+0.0) features, and a pair whose dot cancels to
  zero exactly: the forward equals the oracle bit for bit, signs of zero included; with an integer upstream gradient the
  backward is exact too."""
  rng = np.random.RandomState(F * d)
  feats = rng.randint(-8, 9, size=(B, F, d)).astype(np.float32)
  feats[:, 1] = -feats[:, 0]
  feats[:, 2] = -0.0
  feats[:, 3] = 0.0
  feats[:, 4] = np.where(np.arange(d) % 2 == 0, 1.0, -1.0)
  feats[:, 5] = np.where(np.arange(d) < d - d % 2, 1.0, 0.0)        # e_4 . e_5 = 1 - 1 + 1 - ... = +0 exactly
  feats[:, 6, ::2] = -0.0
  feats[:, 6, 1::2] = 3.0
  x = torch.from_numpy(feats).cuda()
  for si, sg in DI_MODES:
    exp = _di_oracle(feats, si, sg)
    assert np.array_equal(_bits(ops.dot_interaction(x, si, sg)), exp.view(np.int32)), (si, sg)
    g = rng.randint(-4, 5, size=exp.shape).astype(np.float32)
    xg = x.clone().requires_grad_(True)
    ops.dot_interaction(xg, si, sg).backward(torch.from_numpy(g).cuda())
    ref = orc.dot_interaction_grads([feats[:, f] for f in range(F)], g, si, sg)
    assert np.array_equal(xg.grad.cpu().numpy().astype(np.float64), ref), (si, sg)
