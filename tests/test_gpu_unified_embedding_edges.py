"""K8 (UnifiedEmbedding, csrc/unified_embedding.cu) at its edges, bit for bit against a plain reference.

The per-slot reference is restated here in NumPy: bucket ids from the C oracle's SipHash (`uo.hash_bins`), the row
gather, the bag sum in value order from +0 in float32, one division by float32(count) (mean) or sqrt(float32(count))
(sqrtn) with empty bags left at zero, and the backward's bag gradient divided the same way.  The cases reach what the
shapes of tests/test_gpu_unified_embedding.py do not:
  - every row width class: L = dim/4 of 1, non-powers of two (the `item / L` paths) and L > 8 (several passes of the
    forward's row-copy loop, the next chunk's SipHash issued on the first pass only);
  - value counts at 32-value warp edges, and features of very different n in one launch;
  - chunk counts whose sorted() names reorder the columns, with the table cursor carried across features;
  - calls split into several parameter blocks (64 features / 256 slots each), including features of more than 256
    chunks, which are split across blocks;
  - integer and string messages at every decimal length, string length 0-64 and start offset 0-15 through the fused
    kernel, with register and memory messages in one warp;
  - empty-bag runs, one-bag and 100 000-value bags, NumPy and CUDA row splits, non-contiguous and unused gradients;
  - the C ABI's strided outputs (ld > width, col_off > 0) and its argument errors.
"""
import numpy as np
import pytest
import torch

import unified_oracle as uo

pytestmark = pytest.mark.gpu

INT64_MIN, INT64_MAX = -2**63, 2**63 - 1
INT32_MIN, INT32_MAX = -2**31, 2**31 - 1
UE_MAX_FEATURES, UE_MAX_SLOTS = 64, 256        # one parameter block of csrc/unified_embedding.cu
SIP_SHORT = 23                                 # csrc/siphash.cuh: longer messages are hashed from memory


@pytest.fixture(scope="module")
def tfrs():
  import recommenders_b200 as t
  return t


# ---- the reference -----------------------------------------------------------------------------------------------------
def _bag_sums(rows, splits):
  """Per bag, ((0 + r0) + r1) + ... in float32, in value order."""
  lens = np.diff(splits)
  out = np.zeros((len(lens), rows.shape[1]), np.float32)
  short = lens <= 64
  for k in range(int(lens[short].max(initial=0))):
    b = np.nonzero(short & (lens > k))[0]
    out[b] = out[b] + rows[splits[b] + k]
  for b in np.nonzero(~short)[0]:                # long bags: a sequential running sum that starts at +0
    run = np.concatenate([np.zeros((1, rows.shape[1]), np.float32), rows[splits[b]:splits[b + 1]]])
    out[b] = np.cumsum(run, axis=0, dtype=np.float32)[-1]
  return out


def _divisor(lens, combiner):
  c = np.asarray(lens).astype(np.float32)
  return {"sum": np.ones_like(c), "mean": c, "sqrtn": np.sqrt(c)}[combiner]


def _ref_slot(table, flat, salt, splits=None, combiner="mean"):
  """One (feature, chunk) lookup: (bucket ids, output rows)."""
  ids = np.asarray(uo.hash_bins(flat, table.shape[0], salt)).reshape(-1)
  rows = table[ids]
  if splits is None:
    return ids, rows
  lens = np.diff(splits)
  acc = _bag_sums(rows, splits)
  nz = lens > 0
  acc[nz] = acc[nz] / _divisor(lens[nz], combiner)[:, None]
  return ids, acc


def _ref_slot_bwd(g_cols, splits=None, combiner="mean"):
  """The gradient rows of one slot, value by value, from the gradient at the slot's output columns."""
  if splits is None:
    return np.ascontiguousarray(g_cols, np.float32)
  lens = np.diff(splits)
  bag = np.repeat(np.arange(len(lens)), lens)
  return g_cols[bag] / _divisor(lens, combiner)[bag, None]


def _parts(x):
  values, splits = x if isinstance(x, tuple) else (x, None)
  return np.asarray(values).reshape(-1), (None if splits is None else np.asarray(splits, np.int64)), np.shape(values)


def _ref_forward(host, spec, tables, name, combiner):
  """(outputs, {table: bucket ids in feature, chunk, value order})."""
  dim = tables[0].shape[1]
  outs, ids = [], {}
  for feat, chunks in uo.plan(spec, len(tables), name):
    flat, splits, shape = _parts(host[feat])
    out = np.zeros((flat.size if splits is None else len(splits) - 1, len(chunks) * dim), np.float32)
    for _, t, salt, pos in chunks:
      b, r = _ref_slot(tables[t], flat, salt, splits, combiner)
      ids.setdefault(t, []).append(b)
      out[:, pos * dim:(pos + 1) * dim] = r
    outs.append(out if splits is not None else out.reshape(*shape, -1))
  return outs, {t: np.concatenate(v) for t, v in ids.items()}


def _ref_backward(host, spec, num_tables, dim, name, grads, combiner):
  rows = {}
  for (feat, chunks), g in zip(uo.plan(spec, num_tables, name), grads):
    _, splits, _ = _parts(host[feat])
    g = np.asarray(g, np.float32).reshape(-1, len(chunks) * dim)
    for _, t, _, pos in chunks:
      rows.setdefault(t, []).append(_ref_slot_bwd(g[:, pos * dim:(pos + 1) * dim], splits, combiner))
  return {t: np.concatenate(v) for t, v in rows.items()}


# ---- helpers -----------------------------------------------------------------------------------------------------------
def _same(got, exp, what=""):
  got = got.detach().cpu().numpy() if isinstance(got, torch.Tensor) else np.asarray(got)
  exp = np.ascontiguousarray(exp)
  assert got.shape == exp.shape and got.dtype == exp.dtype, (what, got.shape, got.dtype, exp.shape, exp.dtype)
  if got.tobytes() != exp.tobytes():
    np.testing.assert_array_equal(got, exp, err_msg=what)
    raise AssertionError(f"{what}: equal values but different bits (signed zeros or NaN payloads)")


def _layer(name, num_tables, spec, buckets, dim, combiner="mean", seed=0):
  from recommenders_b200.layers.feature_multiplexing import unified_embedding as ue
  torch.manual_seed(seed)
  cfg = ue.UnifiedEmbeddingConfig(buckets_per_table=buckets, dim_per_table=dim, num_tables=num_tables, name=name,
                                  combiner=combiner)
  for f, c in spec:
    cfg.add_feature(f, c)
  return ue.UnifiedEmbedding(cfg)


def _device(host, numpy_splits=False):
  """CUDA tensors for integer values (and row splits unless `numpy_splits`); strings stay NumPy."""
  def dev(v):
    return torch.from_numpy(np.ascontiguousarray(v)).cuda() if isinstance(v, np.ndarray) and v.dtype.kind in "iu" else v
  return {k: ((dev(v[0]), v[1] if numpy_splits else dev(v[1])) if isinstance(v, tuple) else dev(v))
          for k, v in host.items()}


def _node(out):
  """The layer's autograd node behind an output (dense outputs are reshaped views of the node's output)."""
  fn = out.grad_fn
  while fn is not None and not hasattr(fn, "ids"):
    fn = fn.next_functions[0][0]
  return fn


def _groups(chunks):
  """The parameter blocks of one call, restated: [[(feature, chunks of it in the block)]].  A feature goes whole into
  the current block, or into a fresh one when it does not fit; a feature of more than 256 chunks fills the current
  block and continues in fresh ones."""
  groups, cur, ns = [], [], 0
  for k, nc in enumerate(chunks):
    c0 = 0
    while c0 < nc:
      if cur and (len(cur) == UE_MAX_FEATURES or ns == UE_MAX_SLOTS or (nc <= UE_MAX_SLOTS and ns + nc > UE_MAX_SLOTS)):
        groups.append(cur)
        cur, ns = [], 0
      take = min(nc - c0, UE_MAX_SLOTS - ns)
      cur.append((k, take))
      ns += take
      c0 += take
  return groups + ([cur] if cur else [])


def _launches(chunks, pooled):
  """(forward, backward) launches of a call whose features all have values: per block one forward launch, one
  pooling launch when the block holds a pooled slot, and one backward launch."""
  g = _groups(chunks)
  return len(g) + sum(any(pooled[k] for k, _ in grp) for grp in g), len(g)


def _check_layer(tfrs, layer, host, spec, name, combiner, dev=None, seed=0, launches=None, oracle=False):
  """Forward outputs, the bucket ids the autograd node keeps, and each table's (ids, rows) pair after a backward with
  random gradients, all against the reference; optionally the launch counts and the C oracle's forward."""
  dim = layer._config._dim_per_table
  tables = [t.weight.detach().cpu().numpy() for t in layer._tables]
  for t in layer._tables:
    t.pop_sparse_grads()
  dev = _device(host) if dev is None else dev
  torch.cuda.synchronize()
  n0 = tfrs.ops.launch_count()
  outs = layer(dev)
  n1 = tfrs.ops.launch_count()
  exp, exp_ids = _ref_forward(host, spec, tables, name, combiner)
  if oracle:
    c_out, c_ids = uo.forward(host, spec, tables, name, combiner)
    for a, b in zip(c_out, exp):
      _same(a, b, "the C oracle against the restated reference")
    assert c_ids.keys() == exp_ids.keys() and all(np.array_equal(c_ids[t], exp_ids[t]) for t in c_ids)
  assert len(outs) == len(exp)
  for (feat, _), o, e in zip(spec, outs, exp):
    _same(o, e, f"forward output of {feat}")
  node = _node(outs[0])
  assert sorted(node.ids) == sorted(exp_ids)
  for t, ids in node.ids.items():
    _same(ids, exp_ids[t], f"bucket ids of table {t}")
  rng = np.random.default_rng(seed)
  grads = [rng.standard_normal(tuple(o.shape)).astype(np.float32) for o in outs]
  n2 = tfrs.ops.launch_count()
  torch.autograd.backward(outs, [torch.from_numpy(g).cuda() for g in grads])
  n3 = tfrs.ops.launch_count()
  exp_rows = _ref_backward(host, spec, len(tables), dim, name, grads, combiner)
  for t, tab in enumerate(layer._tables):
    pairs = tab.pop_sparse_grads()
    assert len(pairs) == (1 if t in exp_ids else 0), t
    if pairs:
      _same(pairs[0][0], exp_ids[t], f"backward ids of table {t}")
      _same(pairs[0][1], exp_rows[t], f"backward rows of table {t}")
  if launches is not None:
    assert (n1 - n0, n3 - n2) == launches
  return outs


def _splits(lens):
  return np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)


def _words(rng, n, lo=0, hi=40):
  """n random ASCII strings of lo..hi characters, no NUL."""
  lens = rng.integers(lo, hi + 1, size=n)
  chars = rng.integers(33, 127, size=int(lens.sum()), dtype=np.uint8).tobytes().decode()
  cut = _splits(lens)
  return np.array([chars[cut[i]:cut[i + 1]] for i in range(n)])


# ---- 1. row widths -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("combiner", ["mean", "sum", "sqrtn"])
@pytest.mark.parametrize("dim", [4, 8, 12, 20, 28, 32, 36, 60, 64, 128, 132, 1024])
def test_row_widths(tfrs, dim, combiner):
  """L = dim/4 in {1, 2, 3, 5, 7, 8, 9, 15, 16, 32, 33, 256}: powers of two and not, one and several passes of the
  8-item row copy; 3-4 chunks per feature over 3 tables."""
  rng = np.random.default_rng(dim)
  lens = rng.integers(0, 7, size=40)
  lens[[0, 17, 39]] = 0
  host = {"i64": rng.integers(-10**15, 10**15, size=70),
          "i32": rng.integers(INT32_MIN, INT32_MAX, size=(23, 3), dtype=np.int64).astype(np.int32),
          "s": _words(rng, 70),
          "rag": (rng.integers(0, 10**6, size=int(lens.sum())), _splits(lens))}
  spec = [("i64", 3), ("i32", 3), ("s", 4), ("rag", 3)]
  layer = _layer("w", 3, spec, buckets=1009, dim=dim, combiner=combiner, seed=dim)
  outs = _check_layer(tfrs, layer, host, spec, "w", combiner, seed=dim, launches=(2, 1), oracle=True)
  assert [tuple(o.shape) for o in outs] == [(70, 3 * dim), (23, 3, 3 * dim), (70, 4 * dim), (40, 3 * dim)]


# ---- 2. warp edges -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [1, 31, 32, 33, 255, 256, 257, 8191, 8193])
def test_warp_edges(tfrs, n):
  rng = np.random.default_rng(n)
  cuts = np.sort(rng.integers(0, n + 1, size=max(n // 3, 1) - 1))
  host = {"ids": rng.integers(INT64_MIN, INT64_MAX, size=n, dtype=np.int64),
          "s": _words(rng, n, 0, 40),
          "rag": (rng.integers(-10**6, 10**6, size=n), np.concatenate([[0], cuts, [n]]).astype(np.int64))}
  spec = [("ids", 2), ("s", 1), ("rag", 2)]
  _check_layer(tfrs, _layer("warp", 2, spec, buckets=4099, dim=8), host, spec, "warp", "mean", seed=n, launches=(2, 1))


def test_short_and_long_features_in_one_launch(tfrs):
  """n = 1 and n = 100 000 side by side: almost every warp of the short features exits at once."""
  rng = np.random.default_rng(11)
  n = 100_000
  splits = np.concatenate([[0], np.sort(rng.integers(0, n + 1, size=4999)), [n]]).astype(np.int64)
  host = {"one": rng.integers(0, 10**9, size=1), "many": rng.integers(INT64_MIN, INT64_MAX, size=n, dtype=np.int64),
          "bag1": (rng.integers(0, 10, size=1), np.array([0, 1], np.int64)),
          "bags": (rng.integers(0, 10**12, size=n), splits)}
  spec = [("one", 2), ("many", 2), ("bag1", 2), ("bags", 2)]
  _check_layer(tfrs, _layer("sl", 3, spec, buckets=65537, dim=16), host, spec, "sl", "mean", launches=(2, 1))


# ---- 3. chunk counts and table rotation ----------------------------------------------------------------------------------
@pytest.mark.parametrize("num_tables", [1, 3, 7])
def test_chunk_counts_and_table_rotation(tfrs, num_tables):
  """1, 2, 10 and 11 chunks: sorted() puts `_lookup_10` before `_lookup_2`; the table cursor carries across features."""
  rng = np.random.default_rng(num_tables)
  spec = [("a", 1), ("b", 2), ("c", 10), ("d", 11), ("e", 3)]
  cols = {c: pos for c, _, _, pos in uo.plan(spec, num_tables, "cc")[3][1]}
  assert cols[10] < cols[2] and cols[1] < cols[10]
  host = {k: rng.integers(-10**6, 10**6, size=45) for k in "abcd"}
  host["e"] = (rng.integers(0, 100, size=45), _splits([0, 5, 0, 0, 12, 1, 27, 0]))
  layer = _layer("cc", num_tables, spec, buckets=211, dim=12)
  _check_layer(tfrs, layer, host, spec, "cc", "mean", launches=(2, 1), oracle=True)


# ---- 4. launch groups --------------------------------------------------------------------------------------------------
_GROUP_CASES = {
    "64x1": ([1] * 64, []),
    "65x1": ([1] * 65, []),
    "64x4": ([4] * 64, []),
    "64x4+1": ([4] * 64 + [1], []),
    "63x4+5": ([4] * 63 + [5], [62, 63]),
    "100,200": ([100, 200], []),
    "100,200 pooled": ([100, 200], [0, 1]),
    "256": ([256], []),
    "70x3 pooled around the boundary": ([3] * 70, list(range(1, 70, 2))),
    "70x3 pooled before the boundary": ([3] * 70, [0, 5, 63]),
    "300x1": ([1] * 300, [0, 64, 299]),
}


@pytest.mark.parametrize("case", sorted(_GROUP_CASES))
def test_launch_groups(tfrs, case):
  """Calls longer than one parameter block: outputs, one (ids, rows) pair per table in feature, chunk and value order,
  and one forward launch per block (two with pooled slots), one backward launch per block."""
  chunks, pooled_at = _GROUP_CASES[case]
  rng = np.random.default_rng(len(chunks) * 1000 + sum(chunks))
  n, pooled = 24, [k in pooled_at for k in range(len(chunks))]
  host, spec = {}, []
  for k, nc in enumerate(chunks):
    v = rng.integers(-10**9, 10**9, size=n)
    host[f"f{k}"] = (v, _splits(rng.multinomial(n, np.ones(7) / 7))) if pooled[k] else v
    spec.append((f"f{k}", nc))
  assert len(_groups(chunks)) >= (1 if case in ("64x1", "64x4", "256") else 2)
  layer = _layer("g", 3, spec, buckets=101, dim=4)
  _check_layer(tfrs, layer, host, spec, "g", "mean", launches=_launches(chunks, pooled))


# ---- 5. messages through the fused kernel ---------------------------------------------------------------------------------
def _decimal_edges():
  out = [0, INT64_MIN, INT64_MIN + 1, INT64_MAX, INT64_MAX - 1]
  for k in range(19):
    for x in (10**k - 1, 10**k, 10**k + 1):
      out += [x, -x]
  out += [10**9 * 7, 10**18 + 1, 10**9 + 10**18, -(10**18 + 10**9 + 1)]     # zero digits inside the 10^9 pieces
  return [x for x in out if INT64_MIN <= x <= INT64_MAX]


def _string_layout(rng):
  """Random NUL-free byte strings: every length 0..64 starting at every offset 0..15 of the packed buffer (relative to
  its start), with short pad strings between; consecutive lengths put register and memory messages in one warp."""
  items, pos = [], 0
  rand = lambda k: rng.integers(1, 256, size=k, dtype=np.uint8).tobytes()
  for r in range(16):
    for length in range(65):
      pad = (r - pos) % 16
      if pad:
        items.append(rand(pad))
        pos += pad
      items.append(rand(length))
      pos += length
  for length in (1024, 1023, 1025, 1031):                               # long strings between short ones
    items += [rand(length), rand(3)]
  return items


def test_messages(tfrs):
  rng = np.random.default_rng(12)
  ints = np.array(_decimal_edges(), np.int64)
  ints = np.concatenate([ints, rng.integers(INT64_MIN, INT64_MAX, size=300, dtype=np.int64)])
  rng.shuffle(ints)
  i32 = np.array([INT32_MIN, INT32_MIN + 1, INT32_MAX, INT32_MAX - 1, 0, -1, 1] +
                 [s * (10**k + d) for k in range(10) for d in (-1, 0) for s in (1, -1) if 10**k + d <= INT32_MAX],
                 np.int64)
  i32 = np.concatenate([i32, rng.integers(INT32_MIN, INT32_MAX, size=100)]).astype(np.int32)
  items = _string_layout(rng)
  byts = np.empty(len(items), dtype=object)
  byts[:] = items
  text = np.array(["", "é", "日本語", "héllo wörld " * 3, "🙂" * 6, "Zürich", "x" * 24, "ü" * 12, "ü" * 11 + "u"] * 9)
  host = {"ints": ints, "i32": i32, "bytes": byts, "text": text}
  spec = [("ints", 3), ("i32", 3), ("bytes", 4), ("text", 3)]
  layer = _layer("msg", 2, spec, buckets=1_000_003, dim=4)
  dev = _device(host)
  outs = layer(dev)
  node = _node(outs[0])
  # the layout reaches what it is meant to: every (length, start mod 16) of the packed bytes, and mixed warps
  x = node.inputs[2]
  off = x.offsets.cpu().numpy()
  starts, lens = (x.values.data_ptr() + off[:-1]) % 16, np.diff(off)
  for length in range(65):
    assert set(starts[lens == length].tolist()) == set(range(16)), length
  long_ = np.pad(lens > SIP_SHORT, (0, -len(lens) % 32)).reshape(-1, 32)
  assert (long_.any(1) & ~long_.all(1)).sum() > 30
  assert max(len(s.encode()) for s in text) > SIP_SHORT
  del outs, node
  _check_layer(tfrs, layer, host, spec, "msg", "mean", dev=dev, launches=(1, 1), oracle=True)


# ---- 6. pooling and backward -----------------------------------------------------------------------------------------------
def _bag_lengths(rng):
  """Empty bags at the start, in runs in the middle and at the end; every length 1..9."""
  lens = [0, 0, 0] + [k for k in range(1, 10)] + [0] * 5 + list(rng.integers(0, 10, size=60)) + [0, 7, 0, 0, 1, 0] + [0] * 4
  return np.array(lens, np.int64)


@pytest.mark.parametrize("splits_on", ["cuda", "numpy"])
@pytest.mark.parametrize("combiner", ["mean", "sum", "sqrtn"])
def test_pooling_bags(tfrs, combiner, splits_on):
  rng = np.random.default_rng(13)
  lens = _bag_lengths(rng)
  n = int(lens.sum())
  host = {"bags": (rng.integers(-10**6, 10**6, size=n), _splits(lens)),
          "words": (_words(rng, n, 0, 30), _splits(lens)),
          "all_in_one": (rng.integers(0, 10**6, size=50), np.array([0, 0, 50, 50], np.int64)),
          "single_bag": (rng.integers(0, 10**6, size=37), np.array([0, 37], np.int64)),
          "dense": rng.integers(0, 10**6, size=9)}
  spec = [("bags", 2), ("words", 3), ("all_in_one", 2), ("single_bag", 1), ("dense", 2)]
  layer = _layer("pool", 3, spec, buckets=97, dim=8, combiner=combiner)
  dev = _device(host, numpy_splits=splits_on == "numpy")
  if splits_on == "numpy":
    # the NumPy row splits and the strings of a call share one upload
    node_inputs = _node(layer(dev)[0]).inputs
    bases = {x.row_splits.untyped_storage().data_ptr() for x in node_inputs if x.row_splits is not None}
    assert bases == {node_inputs[1].values.untyped_storage().data_ptr()}
  _check_layer(tfrs, layer, host, spec, "pool", combiner, dev=dev, launches=(2, 1), oracle=True)


@pytest.mark.parametrize("combiner", ["mean", "sum", "sqrtn"])
def test_one_long_bag(tfrs, combiner):
  """A 100 000-value bag among short ones: one lane group sums it in order; the backward's binary search finds it."""
  rng = np.random.default_rng(14)
  lens = np.array([0, 3, 100_000, 0, 1, 0], np.int64)
  host = {"long": (rng.integers(INT64_MIN, INT64_MAX, size=int(lens.sum()), dtype=np.int64), _splits(lens))}
  spec = [("long", 2)]
  layer = _layer("long", 2, spec, buckets=50, dim=12, combiner=combiner)
  _check_layer(tfrs, layer, host, spec, "long", combiner, launches=(2, 1))


def _loss_inputs(rng):
  lens = _bag_lengths(rng)
  return {"dense": rng.integers(0, 10**6, size=50), "multi": rng.integers(0, 10**6, size=(20, 4)),
          "bags": (rng.integers(0, 10**6, size=int(lens.sum())), _splits(lens)), "words": _words(rng, 50),
          "unused": rng.integers(0, 10**6, size=50)}


@pytest.mark.parametrize("how", ["views in the loss", "strided gradients"])
def test_noncontiguous_and_unused_gradients(tfrs, how):
  """Outputs sliced, expanded or transposed before the loss, or gradients handed in with strides: the backward takes
  each incoming gradient as it comes; an output left out of the loss gives zero rows."""
  rng = np.random.default_rng(15)
  host = _loss_inputs(rng)
  spec = [("dense", 2), ("multi", 3), ("bags", 2), ("words", 1), ("unused", 2)]
  layer = _layer("nc", 3, spec, buckets=301, dim=8, combiner="sqrtn")
  tables = [t.weight.detach().cpu().numpy() for t in layer._tables]
  outs = layer(_device(host))
  w = [torch.from_numpy(rng.standard_normal((3,) + tuple(o.shape)).astype(np.float32)).cuda() for o in outs]

  def loss(o):
    return ((o[0][:, 3:-5] * w[0][0, :, 3:-5]).sum() + (o[1][:, 1:3].expand(3, -1, -1, -1) * w[1][:, :, 1:3]).sum() +
            (o[2].t()[::2] * w[2][0].t()[::2]).sum() + (o[3].unsqueeze(0).expand(3, -1, -1) * w[3]).sum())

  if how == "views in the loss":
    proxies = [o.detach().clone().requires_grad_() for o in outs]
    loss(proxies).backward()
    grads = [p.grad if p.grad is not None else torch.zeros_like(p) for p in proxies]
    loss(outs).backward()
  else:
    grads = [w[0][0].t().contiguous().t(), w[1][0].transpose(1, 2).contiguous().transpose(1, 2),
             w[2][1, :1].expand_as(outs[2]), torch.cat([w[3][0], w[3][1]], 1)[:, ::2], torch.zeros_like(outs[4])]
    assert not any(g.is_contiguous() for g in grads[:4])
    torch.autograd.backward(outs[:4], grads[:4])
  assert grads[4].abs().sum() == 0
  grads = [g.cpu().numpy() for g in grads]
  _, exp_ids = _ref_forward(host, spec, tables, "nc", "sqrtn")
  exp_rows = _ref_backward(host, spec, 3, 8, "nc", grads, "sqrtn")
  for t, tab in enumerate(layer._tables):
    (ids, rows), = tab.pop_sparse_grads()
    _same(ids, exp_ids[t], f"ids of table {t}")
    _same(rows, exp_rows[t], f"rows of table {t}")


def test_two_calls_before_a_step(tfrs):
  """Each call appends its own (ids, rows) pair per table, in call order."""
  rng = np.random.default_rng(16)
  spec = [("dense", 2), ("multi", 3), ("bags", 2), ("words", 1), ("unused", 2)]
  layer = _layer("two", 4, spec, buckets=301, dim=8)
  tables = [t.weight.detach().cpu().numpy() for t in layer._tables]
  expected = {t: [] for t in range(4)}
  for call in range(2):
    host = _loss_inputs(rng)
    outs = layer(_device(host))
    grads = [rng.standard_normal(tuple(o.shape)).astype(np.float32) for o in outs]
    torch.autograd.backward(outs, [torch.from_numpy(g).cuda() for g in grads])
    _, ids = _ref_forward(host, spec, tables, "two", "mean")
    rows = _ref_backward(host, spec, 4, 8, "two", grads, "mean")
    for t in ids:
      expected[t].append((ids[t], rows[t]))
  for t, tab in enumerate(layer._tables):
    pairs = tab.pop_sparse_grads()
    assert len(pairs) == len(expected[t]) == 2
    for (ids, rows), (ei, er) in zip(pairs, expected[t]):
      _same(ids, ei)
      _same(rows, er)


# ---- 7. the C ABI through ops --------------------------------------------------------------------------------------------
NAN_FILL = np.uint32(0x7FC00123)       # a quiet NaN with a payload: untouched columns keep these bits


def _abi_call(tfrs, rng):
  """One dense and one pooled input; five slots of four widths and four bucket counts writing at column offsets > 0
  into two [rows, 136] outputs (ld > every slot's columns)."""
  ops = tfrs.ops
  n, LD = 77, 136
  lens = rng.multinomial(n, np.ones(20) / 20)
  lens[[0, 7, 8]] = 0
  lens[1] += n - lens.sum()
  splits = _splits(lens)
  values = rng.integers(-10**15, 10**15, size=n)
  tables = {d: rng.standard_normal((r, d)).astype(np.float32) for d, r in ((4, 97), (12, 1009), (64, 13), (8, 4096))}
  tt = {d: torch.from_numpy(t).cuda() for d, t in tables.items()}
  v = torch.from_numpy(values).cuda()
  inputs = [ops.LookupInput(v), ops.LookupInput(v, None, torch.from_numpy(splits).cuda(), "sqrtn")]
  layout = [(0, 4, 4), (0, 12, 16), (0, 64, 48), (1, 8, 8), (1, 64, 68)]      # (input, dim, col_off)
  salts = [(2**64 - 1, 0), (1, 2), (3, 2**63), (12345, 678), (0, 0)]
  return inputs, layout, salts, tables, tt, values, splits, n, LD


def _abi_slots(tfrs, inputs, layout, salts, tt, outs, ids):
  return [tfrs.ops.LookupSlot(k, tt[d], s, outs[k], col, ids[c]) for c, ((k, d, col), s) in enumerate(zip(layout, salts))]


def _filled(shape, rng=None):
  """A CUDA float32 tensor of NAN_FILL bits, or of random bits from `rng`."""
  a = np.full(shape, NAN_FILL, np.uint32) if rng is None else rng.integers(0, 2**32, size=shape, dtype=np.uint32)
  return torch.from_numpy(a.view(np.float32)).cuda()


def test_c_abi_strided_outputs(tfrs):
  ops = tfrs.ops
  rng = np.random.default_rng(17)
  inputs, layout, salts, tables, tt, values, splits, n, LD = _abi_call(tfrs, rng)
  rows_of = [n, len(splits) - 1]
  outs = [_filled((rows_of[0], LD)), _filled((rows_of[1], LD))]
  ids = [torch.full((n,), -7, dtype=torch.int64, device="cuda") for _ in layout]
  ids[1] = None                                             # an unpooled slot may skip its ids
  torch.cuda.synchronize()
  n0 = ops.launch_count()
  ops.unified_lookup(inputs, _abi_slots(tfrs, inputs, layout, salts, tt, outs, ids))
  assert ops.launch_count() - n0 == 2
  exp = [np.full((r, LD), NAN_FILL, np.uint32).view(np.float32) for r in rows_of]
  for c, ((k, d, col), s) in enumerate(zip(layout, salts)):
    b, r = _ref_slot(tables[d], values, s, splits if k else None, "sqrtn")
    exp[k][:, col:col + d] = r
    if ids[c] is not None:
      _same(ids[c], b, f"ids of slot {c}")
  for k in range(2):
    _same(outs[k], exp[k], f"output {k}")            # the columns outside the slots keep their NaN bits
  # garbage in the output beforehand changes no slot column; a repeated call is byte-identical
  garbage = [_filled(o.shape, rng=rng) for o in outs]
  g0 = [g.cpu().numpy().copy() for g in garbage]
  ops.unified_lookup(inputs, _abi_slots(tfrs, inputs, layout, salts, tt, garbage, [None, None, None] + ids[3:]))
  for k in range(2):
    e = g0[k].copy()
    for kk, d, col in layout:
      if kk == k:
        e[:, col:col + d] = exp[k][:, col:col + d]
    _same(garbage[k], e, f"output {k} over garbage")
  again = [o.clone() for o in outs]
  ops.unified_lookup(inputs, _abi_slots(tfrs, inputs, layout, salts, tt, outs, ids))
  for a, b in zip(again, outs):
    assert a.cpu().numpy().tobytes() == b.cpu().numpy().tobytes()
  # the backward reads each slot's gradient columns at the same ld and col_off
  grads = [torch.from_numpy(rng.standard_normal((r, LD)).astype(np.float32)).cuda() for r in rows_of]
  grad_rows = [torch.full((n, d), float("nan"), device="cuda") for _, d, _ in layout]
  n0 = ops.launch_count()
  ops.unified_lookup_bwd(inputs, _abi_slots(tfrs, inputs, layout, salts, tt, outs, ids),
                         [grads[k] for k, _, _ in layout], grad_rows)
  assert ops.launch_count() - n0 == 1
  for c, (k, d, col) in enumerate(layout):
    g = grads[k].cpu().numpy()[:, col:col + d]
    _same(grad_rows[c], _ref_slot_bwd(g, splits if k else None, "sqrtn"), f"gradient rows of slot {c}")


def test_c_abi_argument_errors(tfrs):
  """Each bad argument raises before anything is launched."""
  ops = tfrs.ops
  rng = np.random.default_rng(18)
  inputs, layout, salts, tables, tt, values, splits, n, LD = _abi_call(tfrs, rng)
  outs = [_filled((n, LD)), _filled((len(splits) - 1, LD))]
  ids = [torch.empty(n, dtype=torch.int64, device="cuda") for _ in layout]

  def slots(**change):
    s = _abi_slots(tfrs, inputs, layout, salts, tt, outs, ids)
    c = change.pop("slot", 0)
    s[c] = s[c]._replace(**change)
    return s

  odd = torch.zeros((97, 6), device="cuda")
  flat = torch.zeros(n * LD + 4, device="cuda")
  bad = [slots(table=odd),                                              # dim not a multiple of 4
         slots(col_off=2),                                              # col_off not a multiple of 4
         slots(out=torch.zeros((n, 130), device="cuda")),               # ld not a multiple of 4
         slots(out=flat[1:1 + n * LD].view(n, LD)),                     # output 4 bytes off its 16-byte alignment
         slots(slot=3, ids=None)]                                       # a pooled slot without its ids
  torch.cuda.synchronize()
  n0 = ops.launch_count()
  for s in bad:
    with pytest.raises(ValueError):
      ops.unified_lookup(inputs, s)
  # chunk counts that disagree with n_slots, straight through the C entry point
  for n_slots, extra in ((len(layout) - 1, 0), (len(layout), 1), (len(layout) + 1, 0)):
    s = slots()
    feats, cs = ops._ue_structs(inputs, s, [x.out for x in s])
    for c, x in enumerate(s):
      cs[c].out = x.out.data_ptr()
    feats[1].n_chunks += extra
    with pytest.raises(ValueError, match="chunks"):
      ops.check(ops.lib().tfrs_unified_lookup_fwd_f32(feats, len(inputs), cs, n_slots, ops.stream()), "unified_lookup")
  assert ops.launch_count() == n0
  ops.unified_lookup(inputs, slots())                                  # and the call itself is fine
  assert ops.launch_count() == n0 + 2


# ---- 8. more than 256 chunks in one feature ---------------------------------------------------------------------------------
@pytest.mark.parametrize("pooled", [False, True])
@pytest.mark.parametrize("n_chunks", [257, 300])
def test_more_than_256_chunks(tfrs, n_chunks, pooled):
  """One feature's chunks are split across parameter blocks: each chunk keeps its salt, table and column."""
  rng = np.random.default_rng(n_chunks + pooled)
  v = rng.integers(-10**12, 10**12, size=40)
  host = {"big": (v, _splits([0, 11, 0, 20, 9])) if pooled else v}
  spec = [("big", n_chunks)]
  _check_layer(tfrs, _layer("big", 3, spec, buckets=61, dim=4), host, spec, "big", "mean",
               launches=_launches([n_chunks], [pooled]))


def test_long_features_between_others(tfrs):
  """A 257-chunk feature after a 100-chunk one fills that block; a pooled 300-chunk feature shares blocks with it."""
  rng = np.random.default_rng(19)
  chunks, pooled = [100, 257, 300, 2], [False, False, True, True]
  host, spec = {}, []
  for k, nc in enumerate(chunks):
    v = rng.integers(0, 10**9, size=33)
    host[f"f{k}"] = (v, _splits([3, 0, 30])) if pooled[k] else v
    spec.append((f"f{k}", nc))
  assert [[c for _, c in g] for g in _groups(chunks)] == [[100, 156], [101, 155], [145, 2]]
  _check_layer(tfrs, _layer("mix256", 5, spec, buckets=53, dim=8), host, spec, "mix256", "mean",
               launches=_launches(chunks, pooled))
