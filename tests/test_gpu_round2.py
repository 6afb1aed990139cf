"""Round-2 GPU parity tests (through the C ABI): exclusions fused into the tensor-core finalize, the fused
FactorizedTopK count, Streaming on the tensor-core path (device and host-resident corpora), full-size checks of
BASELINE configs 3/4/5 against the float64 / canonical oracle, and the compile-then-build optimizer order."""
import numpy as np
import pytest
import torch

from oracle import oracle as orc

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ops():
  from recommenders_b200 import ops as o
  return o


def _rand(shape, seed, scale=1.0):
  g = torch.Generator(device="cuda"); g.manual_seed(seed)
  return torch.randn(shape, generator=g, device="cuda") * scale


# ------------------------------------------------------------------------------------------------
# query_with_exclusions (layers/factorized_top_k.py:83-115, 242-288)
# ------------------------------------------------------------------------------------------------
def _exclusions(ei: torch.Tensor, E: int, n_ids: int, seed: int) -> torch.Tensor:
  """per query: some of its true top hits (so the exclusion matters) + random identifiers"""
  g = torch.Generator(device="cuda"); g.manual_seed(seed)
  ex = torch.randint(0, n_ids, (ei.shape[0], E), generator=g, device="cuda")
  ex[:, 0] = ei[:, 0]; ex[:, 1] = ei[:, 3]; ex[:, 2] = ei[:, ei.shape[1] // 2]
  ex[::7, 3] = ei[::7, -1]
  return ex


@pytest.mark.parametrize("Q,N,d,k,E", [(130, 50000, 64, 20, 7), (300, 131072, 64, 100, 5), (64, 70001, 128, 10, 33)])
def test_tc_exclude_default_identifiers(ops, Q, N, d, k, E):
  c = _rand((N, d), 41); q = _rand((Q, d), 42)
  es, ei = ops.topk_scan(q, c, k + E)
  ex = _exclusions(ei, E, N, 43)
  image = ops.index_build(c)
  s, i = ops.topk_tc_exclude(q, c, image, k, ex)
  st = ops.tc_last_call_stats(Q, N, d, k + E)
  assert st["fallback_queries"] == 0, st
  # the reference's rule on the over-fetched exact list (oracle/oracle.py: exclude)
  os_, oi = orc.exclude(es.cpu().numpy(), ei.cpu().numpy(), ex.cpu().numpy(), k)
  np.testing.assert_array_equal(i.cpu().numpy(), oi)
  np.testing.assert_array_equal(s.cpu().numpy().view(np.uint32), os_.view(np.uint32))
  # and from scratch on the CPU for a few rows
  r = 6
  cs, ci = orc.query_with_exclusions(lambda qq, kk: orc.topk_scan(qq, c.cpu().numpy(), kk), q[:r].cpu().numpy(), ex[:r].cpu().numpy(), k)
  np.testing.assert_array_equal(i[:r].cpu().numpy(), ci)
  np.testing.assert_array_equal(s[:r].cpu().numpy(), cs)


def test_tc_exclude_duplicate_identifiers_and_layers(ops):
  """Identifiers that repeat: more than E fetched rows can be excluded, the reference then returns excluded rows at the
  tail with their ORIGINAL scores -- the fused kernel must do exactly the same.  Also the layer-level entry points."""
  import recommenders_b200 as tfrs
  N, d, Q, k, E = 60000, 64, 90, 12, 4
  c = _rand((N, d), 51); q = _rand((Q, d), 52)
  ids = (torch.arange(N, device="cuda") // 3).to(torch.int64) * 10 + 7      # triples share an identifier
  es, ei = ops.topk_scan(q, c, k + E)
  ex = ids[_exclusions(ei, E, N, 53)]
  os_, oid = orc.exclude(es.cpu().numpy(), ids[ei].cpu().numpy(), ex.cpu().numpy(), k)
  layer = tfrs.layers.factorized_top_k.BruteForce(k=k).index(c, ids)
  s, got = layer.query_with_exclusions(q, ex)
  np.testing.assert_array_equal(got.cpu().numpy(), oid)
  np.testing.assert_array_equal(s.cpu().numpy(), os_)
  # the exact CUDA-core path + the standalone re-rank kernel (small corpus)
  small = tfrs.layers.factorized_top_k.BruteForce(k=k).index(c[:3000], ids[:3000])
  es2, ei2 = ops.topk_scan(q, c[:3000], k + E)
  ex2 = ids[_exclusions(ei2, E, 3000, 54)]
  o2s, o2i = orc.exclude(es2.cpu().numpy(), ids[ei2].cpu().numpy(), ex2.cpu().numpy(), k)
  s2, i2 = small.query_with_exclusions(q, ex2)
  np.testing.assert_array_equal(i2.cpu().numpy(), o2i); np.testing.assert_array_equal(s2.cpu().numpy(), o2s)
  # Streaming: carried state over k + E, then the same kernel
  ds = tfrs.data.Dataset.from_tensor_slices((ids, c)).batch(4096)
  st = tfrs.layers.factorized_top_k.Streaming(k=k).index_from_dataset(ds)
  s3, i3 = st.query_with_exclusions(q, ex)
  np.testing.assert_array_equal(i3.cpu().numpy(), oid); np.testing.assert_array_equal(s3.cpu().numpy(), os_)


# ------------------------------------------------------------------------------------------------
# FactorizedTopK: the count inside the scan (metrics/factorized_top_k.py:133-192)
# ------------------------------------------------------------------------------------------------
def test_tc_count_equals_exact_rank(ops):
  N, d, Q, kmax = 100000, 64, 256, 100
  c = _rand((N, d), 61); q = _rand((Q, d), 62)
  es, ei = ops.topk_scan(q, c, kmax)
  true = torch.randint(0, N, (Q,), device="cuda")
  true[:64] = ei[torch.arange(64), torch.arange(64) % 7]          # positives that ARE top hits (exact ties with themselves)
  true[64:96] = ei[torch.arange(64, 96), 99]                      # the boundary of the list
  t_emb = c[true].clone()
  t_emb[96:128] += 0.01 * _rand((32, d), 63)                      # positives that are not corpus rows
  pos = ops.rowwise_dot(q, t_emb)
  pos[128] = float("nan"); pos[129] = float("inf"); pos[130] = -float("inf")
  image = ops.index_build(c)
  cnt = ops.topk_tc_count(q, c, image, kmax, pos)
  st = ops.tc_last_call_stats(Q, N, d, kmax)
  assert st["fallback_queries"] == 0, st
  full = orc.scores(q.cpu().numpy(), c.cpu().numpy())             # canonical chain, [Q, N]
  p = pos.cpu().numpy()
  exp = np.minimum((full > p[:, None]).sum(1), kmax)
  np.testing.assert_array_equal(cnt.cpu().numpy(), exp)
  # the list-based count (exact path / Streaming) agrees
  np.testing.assert_array_equal(ops.count_above(es, pos).cpu().numpy(), exp)


@pytest.mark.parametrize("weighted", [False, True])
def test_factorized_topk_metric_fused_vs_oracle(ops, weighted):
  import recommenders_b200 as tfrs
  N, d, Q = 80000, 64, 300
  ks = (1, 5, 10, 50, 100)
  c = _rand((N, d), 71); q = _rand((Q, d), 72)
  true = torch.randint(0, N, (Q,), device="cuda")
  q[:150] = c[true[:150]] * 0.8 + 0.2 * q[:150]                   # half of the queries are close to their positive
  w = torch.rand((Q,), device="cuda") if weighted else None
  cn = c.cpu().numpy()
  exp = orc.factorized_top_k_update(q.cpu().numpy(), cn[true.cpu().numpy()], lambda qq, kk: orc.topk_scan(qq, cn, kk), ks,
                                    sample_weight=None if w is None else w.cpu().numpy())
  bf = tfrs.layers.factorized_top_k.BruteForce().index(c)
  assert bf._tc_index is not None
  for layer in (bf, tfrs.data.Dataset.from_tensor_slices(c).batch(8192)):
    m = tfrs.metrics.FactorizedTopK(layer, ks=ks)
    m.update_state(q, c[true], sample_weight=w)
    m.update_state(q[:100], c[true[:100]], sample_weight=None if w is None else w[:100])   # a second batch accumulates
    exp2 = orc.factorized_top_k_update(q[:100].cpu().numpy(), cn[true[:100].cpu().numpy()], lambda qq, kk: orc.topk_scan(qq, cn, kk),
                                       ks, sample_weight=None if w is None else w[:100].cpu().numpy())
    for got, (num, den), (num2, den2) in zip(m.result(), exp, exp2):
      assert abs(got - (num + num2) / (den + den2)) < 1e-6
    # id-based branch on the same layer
    mi = tfrs.metrics.FactorizedTopK(layer, ks=ks)
    mi.update_state(q, c[true], true_candidate_ids=true.to(torch.int32), sample_weight=w)
    expi = orc.factorized_top_k_update(q.cpu().numpy(), cn[true.cpu().numpy()], lambda qq, kk: orc.topk_scan(qq, cn, kk), ks,
                                       true_ids=true.cpu().numpy(), sample_weight=None if w is None else w.cpu().numpy())
    for got, (num, den) in zip(mi.result(), expi):
      assert abs(got - num / den) < 1e-6
    m.reset_states()
    assert m.result() == [0.0] * len(ks)


# ------------------------------------------------------------------------------------------------
# Streaming at scale (layers/factorized_top_k.py:404-509)
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("where", ["device", "host", "pinned"])
def test_streaming_tensor_core_chunks(ops, where):
  import recommenders_b200 as tfrs
  N, d, Q, k = 300000, 64, 512, 100
  c = _rand((N, d), 81); q = _rand((Q, d), 82)
  c[250000] = c[17]                                                # an exact tie across chunks: the earlier row wins
  es, ei = ops.topk_scan(q, c, k)
  src = c if where == "device" else c.cpu()
  if where == "pinned":
    src = src.pin_memory()
  ds = tfrs.data.Dataset.from_tensor_slices(src).batch(4096)
  st = tfrs.layers.factorized_top_k.Streaming(k=k).index_from_dataset(ds)
  st._coalesce_rows = 65536                                        # 4 tensor-core chunks + a 37856-row tail
  s, i = st(q)
  assert torch.equal(i.to(torch.int64), ei) and torch.equal(s, es)
  assert int(st._counter) == N
  if where != "device":
    assert st._stager is not None and st._stager.h2d_bytes == N * d * 4
    s2, i2 = st(q)                                                 # the staging buffers are reused
    assert torch.equal(i2.to(torch.int64), ei) and torch.equal(s2, es)
  # identifiers ride along
  ids = torch.arange(N, device="cuda", dtype=torch.int64) * 3 + 1
  ds2 = tfrs.data.Dataset.from_tensor_slices((ids, src)).batch(10000)
  s3, i3 = tfrs.layers.factorized_top_k.Streaming(k=k).index_from_dataset(ds2)(q)
  assert torch.equal(i3, ids[ei]) and torch.equal(s3, es)


# ------------------------------------------------------------------------------------------------
# BASELINE configs at full size
# ------------------------------------------------------------------------------------------------
def test_cfg3_full_size_loss_and_gradients_vs_float64(ops):
  """cfg3: B = C = 16384, d = 64, tensor-core forward + backward against float64 NumPy: loss to 1e-5 relative,
  64 sampled rows of dq and of dc to 1e-5 of the true gradient scale."""
  B, d = 16384, 64
  g = torch.Generator(device="cuda"); g.manual_seed(5)
  q = ((torch.rand((B, d), generator=g, device="cuda") - 0.5) * 0.6).requires_grad_(True)
  c = ((torch.rand((B, d), generator=g, device="cuda") - 0.5) * 0.6).requires_grad_(True)
  w = torch.rand((B,), generator=g, device="cuda")
  temp = 0.5
  loss = ops.inbatch_softmax_loss(q, c, w, temp)
  loss.backward()
  q64 = q.detach().cpu().numpy().astype(np.float64); c64 = c.detach().cpu().numpy().astype(np.float64)
  w64 = w.cpu().numpy().astype(np.float64)
  lse = np.empty(B); diag = np.empty(B)
  for lo in range(0, B, 2048):
    S = (q64[lo:lo + 2048] @ c64.T) / temp
    m = S.max(1); lse[lo:lo + 2048] = m + np.log(np.exp(S - m[:, None]).sum(1)); diag[lo:lo + 2048] = S[np.arange(S.shape[0]), lo + np.arange(S.shape[0])]
  exp_loss = float((w64 * (lse - diag)).sum())
  assert abs(float(loss) - exp_loss) <= 1e-5 * abs(exp_loss), (float(loss), exp_loss)
  rows = np.arange(0, B, B // 64)
  # dq_i = sum_j (p_ij - [i=j]) w_i c_j / T
  P = np.exp((q64[rows] @ c64.T) / temp - lse[rows, None]); P[np.arange(len(rows)), rows] -= 1.0
  edq = (P * w64[rows, None]) @ c64 / temp
  # dc_j = sum_i (p_ij - [i=j]) w_i q_i / T
  Pc = np.exp((q64 @ c64[rows].T) / temp - lse[:, None]); Pc[rows, np.arange(len(rows))] -= 1.0
  edc = (Pc * w64[:, None]).T @ q64 / temp
  for got, ref in ((q.grad[rows], edq), (c.grad[rows], edc)):
    err = np.abs(got.cpu().numpy().astype(np.float64) - ref).max()
    assert err <= 1e-5 * np.abs(ref).max(), (err, np.abs(ref).max())


def test_cfg4_shape_d128_two_shards(ops):
  """cfg4's shape (d = 128, 4096 queries, top-100) on a 2M-row corpus: tensor-core path == exact path == oracle, and the
  2-shard decomposition (local scans with offsets -> packed blocks -> sorted merge) returns the same lists."""
  import recommenders_b200 as tfrs
  N, d, Q, k = 2_000_000, 128, 4096, 100
  c = torch.cat([_rand((500_000, d), 90 + b) for b in range(4)], 0); q = _rand((Q, d), 95)
  image = ops.index_build(c)
  s, i = ops.topk_tc(q, c, image, k)
  st = ops.tc_last_call_stats(Q, N, d, k)
  assert st["fallback_queries"] == 0, st
  es, ei = ops.topk_scan(q[:128], c, k)
  assert torch.equal(i[:128], ei) and torch.equal(s[:128], es)
  os_, oi = orc.topk_scan(q[4090:4093].cpu().numpy(), c.cpu().numpy(), k)
  np.testing.assert_array_equal(i[4090:4093].cpu().numpy(), oi); np.testing.assert_array_equal(s[4090:4093].cpu().numpy(), os_)
  parts = []
  for r in range(2):
    lo, hi = tfrs.layers.factorized_top_k.shard_bounds(N, r, 2)
    img = ops.index_build(c[lo:hi])
    parts.append(ops.topk_tc(q, c[lo:hi], img, k, index_offset=lo))
  ms, mi = ops.topk_merge(torch.stack([p[0] for p in parts]), torch.stack([p[1] for p in parts]), k, sorted_lists=True)
  assert torch.equal(mi, i) and torch.equal(ms, s)


def test_cfg5_cross_full_batch_vs_float64(ops):
  """cfg5: one Cross layer at B = 65536, D = 845 (tensor-core forward and backward): sampled rows of out / dx0 / dx and
  the whole dW / dbias against float64 NumPy, 1e-5 of each tensor's true scale."""
  B, D = 65536, 845
  g = torch.Generator(device="cuda"); g.manual_seed(9)
  x0 = torch.rand((B, D), generator=g, device="cuda").requires_grad_(True)
  x = torch.rand((B, D), generator=g, device="cuda").requires_grad_(True)
  W = (torch.randn((D, D), generator=g, device="cuda") * 0.05).requires_grad_(True)
  b = torch.randn((D,), generator=g, device="cuda").requires_grad_(True)
  gout = torch.randn((B, D), generator=g, device="cuda")
  out = ops.cross(x0, x, W, b, 0.0)
  out.backward(gout)
  rows = np.arange(0, B, B // 64)
  x0n = x0.detach().cpu().numpy().astype(np.float64); xn = x.detach().cpu().numpy().astype(np.float64)
  Wn = W.detach().cpu().numpy().astype(np.float64); bn = b.detach().cpu().numpy().astype(np.float64)
  gn = gout.cpu().numpy().astype(np.float64)
  prod = xn[rows] @ Wn + bn
  eout = x0n[rows] * prod + xn[rows]
  gp_rows = gn[rows] * x0n[rows]
  edx0 = gn[rows] * prod
  edx = gp_rows @ Wn.T + gn[rows]
  gp = gn * x0n
  edW = xn.T @ gp
  edb = gp.sum(0)
  for name, got, ref in (("out", out[rows], eout), ("dx0", x0.grad[rows], edx0), ("dx", x.grad[rows], edx), ("dW", W.grad, edW),
                         ("db", b.grad, edb)):
    err = np.abs(got.detach().cpu().numpy().astype(np.float64) - ref).max()
    assert err <= 1e-5 * np.abs(ref).max(), (name, err, np.abs(ref).max())


# ------------------------------------------------------------------------------------------------
# compile() before the first batch: lazily built Cross weights must still be trained (models/base.py:77-78)
# ------------------------------------------------------------------------------------------------
def test_compile_then_fit_trains_lazily_built_cross():
  import recommenders_b200 as tfrs

  class Ranker(tfrs.Model):
    def __init__(self):
      super().__init__()
      self.emb = tfrs.layers.embedding.Embedding(50, 16)
      self.cross = tfrs.layers.dcn.Cross()
      self.mlcn = tfrs.layers.feature_interaction.MultiLayerDCN(projection_dim=4, num_layers=2)

    def compute_loss(self, inputs, training=False):
      ids, y = inputs
      h = self.mlcn(self.cross(self.emb(ids)))
      return ((h.sum(1) - y) ** 2).mean()

  torch.manual_seed(0)
  model = Ranker()
  model.compile(optimizer=tfrs.optimizers.Adagrad(0.1))            # Keras order: compile, THEN the first batch builds the layers
  ids = torch.randint(0, 50, (64,), device="cuda"); y = torch.randn(64, device="cuda")
  l0 = float(model.train_step((ids, y))["loss"])
  k0 = model.cross.kernel.detach().clone(); u0 = model.mlcn.u_kernels[0].detach().clone(); e0 = model.emb.weight.clone()
  for _ in range(5):
    out = model.train_step((ids, y))
  assert not torch.equal(model.cross.kernel.detach(), k0), "Cross.kernel was never updated"
  assert not torch.equal(model.mlcn.u_kernels[0].detach(), u0) and not torch.equal(model.emb.weight, e0)
  assert float(out["loss"]) < l0


# ------------------------------------------------------------------------------------------------
# sparse Adagrad: rank sort + long runs (hot ids of a Zipf batch) stay bit-exact
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n,rows,d,kind", [(16384, 5, 64, "uniform"), (16384, 1_000_000, 64, "zipf"), (9000, 50000, 32, "zipf"),
                                           (16384, 10_000_000, 64, "uniform"), (40000, 1000, 16, "zipf"), (3000, 7, 200, "uniform")])
def test_sparse_adagrad_hot_ids_bit_exact(ops, n, rows, d, kind):
  rng = np.random.RandomState(n + d)
  if kind == "zipf":
    ids = np.minimum(rng.zipf(1.05, size=n) - 1, rows - 1).astype(np.int64)
  else:
    ids = rng.randint(0, rows, size=n).astype(np.int64)
  ids[::97] = -1 if n > 5000 else ids[::97]            # out-of-range ids are skipped
  used = np.unique(ids[ids >= 0])
  table_rows = int(min(rows, 200_000))                   # keep the host copy small: remap ids into a compact table
  remap = {int(v): j for j, v in enumerate(used)} if rows > table_rows else None
  if remap is not None:
    ids = np.array([remap[int(v)] if v >= 0 else -1 for v in ids], np.int64)
  table = rng.uniform(-0.05, 0.05, size=(table_rows, d)).astype(np.float32)
  acc = np.full((table_rows, d), 0.1, np.float32)
  g = (rng.normal(size=(n, d)) * 0.01).astype(np.float32)
  et, ea = orc.sparse_adagrad(table, acc, ids, g, 0.5)
  tt = torch.from_numpy(table).cuda(); ta = torch.from_numpy(acc).cuda()
  ops.sparse_adagrad_(tt, ta, torch.from_numpy(ids).cuda(), torch.from_numpy(g).cuda(), 0.5)
  np.testing.assert_array_equal(tt.cpu().numpy().view(np.uint32), et.view(np.uint32))
  np.testing.assert_array_equal(ta.cpu().numpy().view(np.uint32), ea.view(np.uint32))
