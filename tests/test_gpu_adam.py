"""GPU tests of K10 (Adam, csrc/adam.cu) and `optimizers.Adam`: the sparse and the dense multi-tensor kernels bit-exact
against the fp32 restatement in tests/adam_oracle.py, determinism, and training through `Model.compile`,
`CompositeOptimizer`, `experimental.models.Ranking` and `UnifiedEmbedding`.  Run with -m gpu."""
import os
import sys

import numpy as np
import pytest
import torch

from oracle import oracle as orc

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import adam_oracle as ao  # noqa: E402

pytestmark = pytest.mark.gpu


def cu(a):
  return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def bits(a):
  return np.ascontiguousarray(a, np.float32).view(np.uint32)


def host(t):
  return t.detach().cpu().numpy()


@pytest.fixture(scope="module")
def tfrs():
  import recommenders_b200 as t
  return t


@pytest.fixture(scope="module")
def ops():
  from recommenders_b200 import ops as o
  return o


# ------------------------------------------------------------------------------------------------
# sparse kernel
# ------------------------------------------------------------------------------------------------
def _rows(d):
  return max(65, min(100_000, 2_000_000 // d)) | 1   # odd: the touched-row bitmap has a partial last word


def _ids(rng, n, rows, kind):
  """Uniform ids, or Zipf ids whose hot ids own runs far longer than 64 (the CTA-per-run kernel); -1 and `rows` are
  planted as out-of-range ids."""
  ids = np.minimum(rng.zipf(1.05, size=n) - 1, rows - 1) if kind == "zipf" else rng.randint(0, rows, size=n)
  ids = ids.astype(np.int64)
  if n > 1:
    ids[::97] = -1
    ids[5::101] = rows
  return ids


def _run_sparse_steps(ops, n, d, kind, id_dtype, lazy, seed, steps=3, lr=0.01):
  """`steps` consecutive steps with fresh ids and gradients, the slots starting from nonzero state so that untouched
  rows decay; every step is compared bit for bit on table, m and v."""
  rng = np.random.RandomState(seed)
  rows = _rows(d)
  x = rng.uniform(-0.05, 0.05, size=(rows, d)).astype(np.float32)
  m = (rng.normal(size=(rows, d)) * 1e-3).astype(np.float32)
  v = rng.uniform(0, 1e-5, size=(rows, d)).astype(np.float32)
  tx, tm, tv = cu(x), cu(m), cu(v)
  for t in range(1, steps + 1):
    ids = _ids(rng, n, rows, kind)
    g = (rng.normal(size=(n, d)) * 0.01).astype(np.float32)
    ops.sparse_adam_(tx, tm, tv, cu(ids.astype(id_dtype)), cu(g), ops.adam_alpha(lr, 0.9, 0.999, t), 0.9, 0.999, 1e-7,
                     lazy=lazy)
    x, m, v = ao.adam_sparse(x, m, v, ids, g, lr, t, lazy=lazy)
    for name, got, want in (("table", tx, x), ("m", tm, m), ("v", tv, v)):
      np.testing.assert_array_equal(bits(host(got)), bits(want), err_msg=f"{name} after step {t}")
  return x, m, v


_DIMS = (1, 3, 8, 32, 64, 100, 129, 1024)
_SPARSE = ([(16384, d, kind, lazy) for d in _DIMS for kind in ("uniform", "zipf") for lazy in (False, True)] +
           [(n, d, kind, lazy) for n in (0, 1, 100_000) for d in (3, 64) for kind in ("uniform", "zipf")
            for lazy in (False, True) if n > 1 or kind == "uniform"])


@pytest.mark.parametrize("n,d,kind,lazy", _SPARSE)
def test_sparse_adam_bit_exact(ops, n, d, kind, lazy):
  """The rank-sort (n <= 16384) and bitonic (n > 16384) grouping, runs longer than 64 members (Zipf), the float4 and the
  scalar decay pass (d % 4), I32 and I64 ids, an empty batch (every row still decays unless lazy)."""
  id_dtype = np.int32 if (n + d + int(lazy)) % 2 else np.int64
  _run_sparse_steps(ops, n, d, kind, id_dtype, lazy, seed=n + d)


@pytest.mark.parametrize("id_dtype", [np.int32, np.int64])
def test_sparse_adam_id_dtypes_and_lazy_rows(ops, id_dtype):
  """Both id types on the same batch; with lazy=True, rows no id touched keep their bits."""
  rng = np.random.RandomState(7)
  rows, d = 1001, 16
  x = rng.uniform(-0.05, 0.05, size=(rows, d)).astype(np.float32)
  m = (rng.normal(size=(rows, d)) * 1e-3).astype(np.float32); v = rng.uniform(0, 1e-5, size=(rows, d)).astype(np.float32)
  ids = np.array([0, 5, 5, -1, rows, rows - 1, 5, 900], np.int64)
  g = rng.normal(size=(ids.size, d)).astype(np.float32)
  tx, tm, tv = cu(x), cu(m), cu(v)
  ops.sparse_adam_(tx, tm, tv, cu(ids.astype(id_dtype)), cu(g), ops.adam_alpha(0.01, 0.9, 0.999, 1), 0.9, 0.999, 1e-7,
                   lazy=True)
  other = np.setdiff1d(np.arange(rows), [0, 5, rows - 1, 900])
  for got, was in ((tx, x), (tm, m), (tv, v)):
    assert np.array_equal(bits(host(got)[other]), bits(was[other]))
  ex, em, ev = ao.adam_sparse(x, m, v, ids, g, 0.01, 1, lazy=True)
  for got, want in ((tx, ex), (tm, em), (tv, ev)):
    np.testing.assert_array_equal(bits(host(got)), bits(want))


def test_sparse_adam_deterministic(ops):
  """Two identical Zipf runs give identical bits (both groupings, lazy or not)."""
  for n, lazy in ((16384, False), (100_000, False), (100_000, True)):
    rng = np.random.RandomState(11)
    rows, d = 20_001, 64
    x = rng.uniform(-0.05, 0.05, size=(rows, d)).astype(np.float32)
    ids = cu(_ids(rng, n, rows, "zipf")); g = cu((rng.normal(size=(n, d)) * 0.01).astype(np.float32))
    outs = []
    for _ in range(2):
      tx, tm, tv = cu(x), torch.zeros((rows, d), device="cuda"), torch.zeros((rows, d), device="cuda")
      for t in (1, 2):
        ops.sparse_adam_(tx, tm, tv, ids, g, ops.adam_alpha(0.01, 0.9, 0.999, t), 0.9, 0.999, 1e-7, lazy=lazy)
      outs.append([bits(host(a)) for a in (tx, tm, tv)])
    for a, b in zip(*outs):
      assert np.array_equal(a, b)


# ------------------------------------------------------------------------------------------------
# dense multi-tensor kernel
# ------------------------------------------------------------------------------------------------
def test_dense_adam_bit_exact_many_variables(ops):
  """More variables than one launch's parameters hold (several launches), numels 0, 1, 1023, 1025 and about 3M."""
  rng = np.random.RandomState(3)
  sizes = [(0,), (1,), (1023,), (1025,), (3_000_017,), (845, 512)] + [(int(s),) for s in rng.randint(1, 40, size=1000)]
  sizes += [(0,), (7, 5)]
  xs = [rng.uniform(-0.5, 0.5, size=s).astype(np.float32) for s in sizes]
  ms = [(rng.normal(size=s) * 1e-2).astype(np.float32) for s in sizes]
  vs = [rng.uniform(0, 1e-3, size=s).astype(np.float32) for s in sizes]
  tx, tm, tv = [cu(a) for a in xs], [cu(a) for a in ms], [cu(a) for a in vs]
  for t in (1, 2):
    gs = [(rng.normal(size=s) * 0.05).astype(np.float32) for s in sizes]
    ops.adam_dense_(tx, [cu(g) for g in gs], tm, tv, ops.adam_alpha(0.003, 0.9, 0.999, t), 0.9, 0.999, 1e-7)
    for i in range(len(sizes)):
      xs[i], ms[i], vs[i] = ao.adam_dense(xs[i], ms[i], vs[i], gs[i], 0.003, t)
      for name, got, want in (("var", tx[i], xs[i]), ("m", tm[i], ms[i]), ("v", tv[i], vs[i])):
        np.testing.assert_array_equal(bits(host(got)), bits(want), err_msg=f"{name} of variable {i}, step {t}")


# ------------------------------------------------------------------------------------------------
# errors
# ------------------------------------------------------------------------------------------------
def test_adam_argument_errors(ops):
  t = torch.zeros((10, 4), device="cuda"); m = torch.zeros_like(t); v = torch.zeros_like(t)
  ids = torch.zeros((2,), dtype=torch.int64, device="cuda"); g = torch.zeros((2, 4), device="cuda")
  rule = dict(alpha=1e-3, beta_1=0.9, beta_2=0.999, epsilon=1e-7)
  with pytest.raises(RuntimeError, match="CUDA"):
    ops.sparse_adam_(t.cpu(), m, v, ids, g, **rule)
  with pytest.raises(RuntimeError, match="CUDA"):
    ops.sparse_adam_(t, m, v, ids.cpu(), g, **rule)
  with pytest.raises(RuntimeError, match="CUDA"):
    ops.adam_dense_([t.cpu()], [g.cpu()], [m.cpu()], [v.cpu()], **rule)
  with pytest.raises(ValueError, match="grad_rows"):
    ops.sparse_adam_(t, m, v, ids, g[:1], **rule)
  with pytest.raises(ValueError, match="m must be"):
    ops.sparse_adam_(t, m[:5], v, ids, g, **rule)
  with pytest.raises(ValueError, match="v must be"):
    ops.sparse_adam_(t, m, torch.zeros((10, 5), device="cuda"), ids, g, **rule)
  with pytest.raises(ValueError, match="same length"):
    ops.adam_dense_([t], [g], [m], [], **rule)
  with pytest.raises(ValueError, match="shape"):
    ops.adam_dense_([t], [t], [m[:3]], [v], **rule)
  with pytest.raises(ValueError, match="contiguous"):
    ops.adam_dense_([t], [t], [m.t()], [v], **rule)
  # limits checked by the library, reported across the ABI
  wide = torch.zeros((3, 1025), device="cuda")
  with pytest.raises(ValueError, match="d=1025"):
    ops.sparse_adam_(wide, torch.zeros_like(wide), torch.zeros_like(wide), ids, torch.zeros((2, 1025), device="cuda"),
                     **rule)
  n = 1 << 24
  t1 = torch.zeros((4, 1), device="cuda")
  with pytest.raises(ValueError, match="2\\^24"):
    ops.sparse_adam_(t1, torch.zeros_like(t1), torch.zeros_like(t1), torch.zeros((n,), dtype=torch.int32, device="cuda"),
                     torch.zeros((n, 1), device="cuda"), **rule)
  assert torch.count_nonzero(t1) == 0


# ------------------------------------------------------------------------------------------------
# the optimizer class, end to end
# ------------------------------------------------------------------------------------------------
def test_two_tower_model_trains_with_adam(tfrs):
  """test_two_tower_model_trains_with_clippy_adagrad with Adam: the CUDA step tracks the oracle step by step.  Adam's
  first steps move an element by about lr * g / (|g| + eps'), whatever the size of g, so the last-bit differences of
  the fp32 gradients would show up as large differences on the few elements with |g| near eps'.  The test therefore
  checks the loss and the gradient rows the tables receive against the float64 oracle, and the update made from those
  rows bit for bit."""
  torch.manual_seed(0)
  rng = np.random.RandomState(42)
  U, I, d, B, lr = 2000, 2000, 64, 4096, 0.01

  class TwoTower(tfrs.Model):

    def __init__(self):
      super().__init__()
      self.user_model = tfrs.layers.embedding.Embedding(U, d)
      self.item_model = tfrs.layers.embedding.Embedding(I, d)
      self.task = tfrs.tasks.Retrieval()

    def compute_loss(self, features, training=False):
      return self.task(self.user_model(features["user_id"]), self.item_model(features["movie_id"]),
                       compute_metrics=not training)

  model = TwoTower()
  opt = tfrs.optimizers.Adam(lr)
  model.compile(optimizer=opt)
  received = {}
  for emb in (model.user_model, model.item_model):   # record the (ids, rows) pairs the optimizer takes

    def spy(emb=emb, pop=emb.pop_sparse_grads):
      pairs = pop()
      received[id(emb)] = [(host(i).reshape(-1), host(g)) for i, g in pairs]
      return pairs
    emb.pop_sparse_grads = spy
  state = {id(e): [host(e.weight).copy(), np.zeros((e.input_dim, d), np.float32), np.zeros((e.input_dim, d), np.float32)]
           for e in (model.user_model, model.item_model)}
  losses = []
  uid = rng.randint(0, U, size=B).astype(np.int64); iid = rng.randint(0, I, size=B).astype(np.int64)
  for step in range(1, 4):
    ut, it = state[id(model.user_model)][0], state[id(model.item_model)][0]
    out = model.train_step({"user_id": cu(uid), "movie_id": cu(iid)})
    losses.append(float(out["loss"]))
    qe, ce = orc.gather(ut, uid), orc.gather(it, iid)
    np.testing.assert_allclose(losses[-1], orc.retrieval_loss(qe, ce), rtol=1e-5)
    dq, dc = orc.retrieval_loss_grads(qe, ce)
    for emb, ids, want in ((model.user_model, uid, dq), (model.item_model, iid, dc)):
      (got_ids, got_rows), = received[id(emb)]
      assert np.array_equal(got_ids, ids)
      np.testing.assert_allclose(got_rows, want, rtol=1e-4, atol=1e-5 * np.abs(want).max())
      x, m, v = state[id(emb)]
      state[id(emb)] = ao.adam_sparse(x, m, v, got_ids, got_rows, lr, step)
      for got, exp in zip((emb.weight, emb._tfrs_adam_m, emb._tfrs_adam_v), state[id(emb)]):
        np.testing.assert_array_equal(bits(host(got)), bits(exp), err_msg=f"step {step}")
  assert losses[-1] < losses[0], losses
  assert opt.iterations == 3 and len(opt.variables()) == 4


class _Tiny(torch.nn.Module):

  def __init__(self, tfrs):
    super().__init__()
    self.emb1 = tfrs.layers.embedding.Embedding(1000, 16)
    self.emb2 = tfrs.layers.embedding.Embedding(300, 8)
    self.w = torch.nn.Parameter(torch.randn((16, 8), device="cuda") * 0.1)
    self.b = torch.nn.Parameter(torch.zeros((8,), device="cuda"))


def _copy(tfrs, src):
  dst = _Tiny(tfrs)
  with torch.no_grad():
    for a, b in ((dst.emb1.weight, src.emb1.weight), (dst.emb2.weight, src.emb2.weight), (dst.w, src.w), (dst.b, src.b)):
      a.copy_(b)
  return dst


def _feed(model, step):
  g = torch.Generator(device="cuda"); g.manual_seed(step)
  for emb, n in ((model.emb1, 700), (model.emb2, 300)):
    ids = torch.randint(0, emb.input_dim, (n,), generator=g, device="cuda")
    rows = torch.randn((n, emb.output_dim), generator=g, device="cuda") * 0.1
    emb._sparse_grads += [(ids[:n // 2], rows[:n // 2]), (ids[n // 2:], rows[n // 2:])]   # two lookups of one table
  model.w.grad = torch.randn(model.w.shape, generator=g, device="cuda") * 0.1
  model.b.grad = torch.randn(model.b.shape, generator=g, device="cuda") * 0.1


@pytest.mark.parametrize("lazy", [False, True])
def test_composite_optimizer_with_adam_matches_its_parts(tfrs, lazy):
  """composite_optimizer_test.py:28-86 for the (Adam: tables, Adagrad: dense) pair, 10 steps."""
  torch.manual_seed(0)
  CompositeOptimizer = tfrs.experimental.optimizers.CompositeOptimizer
  a = _Tiny(tfrs); b = _copy(tfrs, a)
  c1, c2 = tfrs.optimizers.Adam(0.02, lazy_embeddings=lazy), tfrs.optimizers.Adagrad(0.1)
  comp = CompositeOptimizer([(c1, lambda: [a.emb1, a.emb2._anchor]), (c2, lambda: [a.w, a.b])]).bind(a)
  s1, s2 = tfrs.optimizers.Adam(0.02, lazy_embeddings=lazy), tfrs.optimizers.Adagrad(0.1)
  first = a.emb1.weight.clone()
  for step in range(10):
    comp.zero_grad()
    _feed(a, step); _feed(b, step)
    comp.apply_gradients()
    s1.apply_gradients([b.emb1, b.emb2]); s2.apply_gradients([b.w, b.b])
    for x, y in ((a.emb1.weight, b.emb1.weight), (a.emb2.weight, b.emb2.weight), (a.w, b.w), (a.b, b.b)):
      assert torch.equal(x.detach().view(torch.int32), y.detach().view(torch.int32)), step
  assert comp.iterations == 10 and c1.iterations == 10 and len(comp.variables()) == 2 * 2 + 2
  assert not torch.equal(first, a.emb1.weight)
  # the composite's Adam state equals the standalone optimizer's
  for p, q in zip(c1.variables(), s1.variables()):
    assert torch.equal(p.view(torch.int32), q.view(torch.int32))


def _synthetic_data(num_dense, vocab_sizes, dataset_size, batch_size, seed=0):
  """experimental/models/ranking_test.py:_generate_synthetic_data: labels = int((mean(dense) + sum(ids)/sum(vocab)) / 2 + 0.5)."""
  g = torch.Generator(device="cuda"); g.manual_seed(seed)
  dense = torch.rand((dataset_size, num_dense), generator=g, device="cuda")
  sparse = [torch.randint(0, v, (dataset_size,), generator=g, device="cuda", dtype=torch.int32) for v in vocab_sizes]
  labels = ((dense.mean(1) + torch.stack(sparse, -1).sum(1).float() / sum(vocab_sizes)) / 2.0 + 0.5).to(torch.int32)
  return [({"dense_features": dense[lo:lo + batch_size],
            "sparse_features": {str(i): s[lo:lo + batch_size] for i, s in enumerate(sparse)}}, labels[lo:lo + batch_size])
          for lo in range(0, dataset_size - batch_size + 1, batch_size)]


class _ConcatCross(torch.nn.Module):
  """tf.keras.Sequential([Concatenate(), Cross()])."""

  def __init__(self, tfrs):
    super().__init__()
    self.cross = tfrs.layers.feature_interaction.Cross()

  def forward(self, inputs):
    return self.cross(torch.cat(inputs, dim=1))


@pytest.mark.parametrize("interaction", ["dot", "cross"])
def test_ranking_model_trains_with_adam(tfrs, interaction):
  """ranking_test.py:148 compiles the Ranking model with Adam."""
  vocab = [30, 3, 26]
  torch.manual_seed(1)
  model = tfrs.experimental.models.Ranking(
      embedding_layer=torch.nn.ModuleDict({str(i): tfrs.layers.embedding.Embedding(v, 16) for i, v in enumerate(vocab)}),
      feature_interaction=tfrs.layers.feature_interaction.DotInteraction() if interaction == "dot" else _ConcatCross(tfrs))
  model.compile(optimizer=tfrs.optimizers.Adam(0.01))
  data = _synthetic_data(8, vocab, 64, 16, seed=5)
  losses = [float(model.evaluate(data)["loss"])]
  for _ in range(15):
    model.fit(data, epochs=1)
    losses.append(float(model.evaluate(data)["loss"]))
  assert np.isfinite(losses).all() and losses[-1] < losses[0], losses
  metrics = model.evaluate(data, return_dict=True)
  assert "accuracy" in metrics and 0.0 <= metrics["accuracy"] <= 1.0
  assert model.optimizer.iterations == 15 * len(data)
  for p in model.parameters():
    assert torch.isfinite(p).all()


def test_unified_embedding_model_trains_with_adam(tfrs):
  """The uet tutorial's model with Adam: several features share each table, so a table's gradient rows in a step come
  from several features' values; the first step equals the oracle on them."""
  from recommenders_b200.layers.feature_multiplexing import unified_embedding as ue_mod
  torch.manual_seed(0)
  names = ["movie_id", "user_id", "user_gender", "user_zip_code", "user_occupation_text", "bucketized_user_age"]
  cfg = ue_mod.UnifiedEmbeddingConfig(buckets_per_table=500, dim_per_table=8, num_tables=2, name="unified_table")
  for n in names:
    cfg.add_feature(n, 2)
  ue = ue_mod.UnifiedEmbedding(cfg, None)

  class UnifiedEmbeddingModel(tfrs.models.Model):
    def __init__(self):
      super().__init__()
      self.embedding = ue
      self.network = tfrs.layers.blocks.MLP([128, 64, 1], final_activation="sigmoid")
      self.task = tfrs.tasks.Ranking(metrics=[tfrs.metrics.AUC(name="AUC")])

    def compute_loss(self, inputs, training=False):
      feats, labels = inputs
      return self.task(labels, self.network(torch.cat(self.embedding(feats), -1)))

  rng = np.random.default_rng(5)
  data = []
  for _ in range(50):
    uid, mid = rng.integers(0, 200, size=256), rng.integers(0, 300, size=256)
    feats = {"movie_id": np.char.mod("%d", mid), "user_id": np.char.mod("%d", uid),
             "user_gender": np.where(uid % 2 == 0, "True", "False"), "user_zip_code": np.char.mod("%05d", uid * 37 % 1000),
             "user_occupation_text": np.array(["doctor", "artist", "student", "other"])[uid % 4],
             "bucketized_user_age": np.char.mod("%d", 18 + uid % 5 * 7)}
    data.append((feats, torch.from_numpy(((uid + mid) % 3 == 0).astype(np.float32)).cuda().reshape(-1, 1)))
  opt = tfrs.optimizers.Adam(0.003)
  model = UnifiedEmbeddingModel()
  model.compile(optimizer=opt)
  # step 1 by hand, to see the gradients the tables receive
  opt.zero_grad()
  model.compute_loss(data[0], training=True).backward()
  before = [host(t.weight) for t in ue._tables]
  pairs = [[(host(i).reshape(-1), host(g)) for i, g in t._sparse_grads] for t in ue._tables]
  assert all(sum(i.size for i, _ in p) > 256 for p in pairs)   # the values of several features per table
  opt.apply_gradients()
  for t, w, p in zip(ue._tables, before, pairs):
    ids = np.concatenate([i for i, _ in p]); g = np.concatenate([r.reshape(-1, w.shape[1]) for _, r in p])
    ex, em, ev = ao.adam_sparse(w, np.zeros_like(w), np.zeros_like(w), ids, g, 0.003, 1)
    np.testing.assert_array_equal(bits(host(t.weight)), bits(ex))
    np.testing.assert_array_equal(bits(host(t._tfrs_adam_m)), bits(em))
    np.testing.assert_array_equal(bits(host(t._tfrs_adam_v)), bits(ev))
  losses = [float(model.train_step(b)["loss"]) for b in data]
  assert np.isfinite(losses).all()
  assert np.mean(losses[-5:]) < np.mean(losses[:5]), losses
  assert all(t._sparse_grads == [] for t in ue._tables)
  assert opt.iterations == 51
