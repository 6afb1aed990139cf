"""GPU tests of K12 (FTRL, csrc/ftrl.cu) and `optimizers.Ftrl`: the sparse and the dense multi-tensor kernels bit-exact
against the fp32 restatement in tests/ftrl_oracle.py (inside a derived bar for the fp64-pow power mode), determinism,
argument errors, and training through `CompositeOptimizer`, `TPUEmbedding`, `UnifiedEmbedding` and
`experimental.models.Ranking`.  Run with -m gpu."""
import itertools
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import ftrl_oracle as fo  # noqa: E402

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


# The optimizer's arguments (tests/ftrl_oracle.py names); l1 > 0 everywhere, so exact zeros occur.
_RULES = {
    "sqrt": dict(lr=0.05, lr_power=-0.5, l1=0.02, l2=0.01),
    "sqrt_shrink_beta": dict(lr=0.05, lr_power=-0.5, l1=0.02, l2=0.01, l2_shrinkage=0.3, beta=0.5),
    "const": dict(lr=0.05, lr_power=0.0, l1=0.02, l2=0.01),
    "const_shrink_beta": dict(lr=0.05, lr_power=0.0, l1=0.02, l2=0.01, l2_shrinkage=0.3, beta=0.5),
}


def _op_rule(ops, kw):
  """The ops-level scalars of an oracle rule."""
  return dict(lr=kw["lr"], lr_power=kw["lr_power"], l1=kw["l1"], l2a=ops.ftrl_l2(kw["l2"], kw.get("beta", 0.0), kw["lr"]),
              l2_shrinkage=kw.get("l2_shrinkage", 0.0))


def _rows(d):
  return max(65, min(100_000, 2_000_000 // d))


def _ids(rng, n, rows, kind):
  """Uniform ids, or Zipf ids whose hot ids own runs far longer than 64 (the CTA-per-run kernel); -1 and `rows` are
  planted as out-of-range ids."""
  ids = np.minimum(rng.zipf(1.05, size=n) - 1, rows - 1) if kind == "zipf" else rng.randint(0, rows, size=n)
  ids = ids.astype(np.int64)
  if n > 1:
    ids[::97] = -1
    ids[5::101] = rows
  return ids


def _state(rng, shape):
  x = rng.uniform(-0.05, 0.05, size=shape).astype(np.float32)
  a = rng.uniform(0.05, 0.5, size=shape).astype(np.float32)
  z = rng.uniform(-0.05, 0.05, size=shape).astype(np.float32)
  return x, a, z


# ------------------------------------------------------------------------------------------------
# sparse kernel
# ------------------------------------------------------------------------------------------------
_DIMS = (1, 3, 8, 32, 64, 100, 129, 1024)
_SPARSE = ([(16384, d, kind, rule) for d in _DIMS for kind in ("uniform", "zipf") for rule in sorted(_RULES)] +
           [(n, d, kind, rule) for n in (0, 1, 100_000) for d in (3, 64) for kind in ("uniform", "zipf")
            for rule in ("sqrt_shrink_beta", "const") if n > 1 or kind == "uniform"])


@pytest.mark.parametrize("n,d,kind,rule", _SPARSE)
def test_sparse_ftrl_bit_exact(ops, n, d, kind, rule):
  """Three steps with fresh ids and gradients, bit for bit on table, accum and linear: the rank-sort (n <= 16384) and
  bitonic (n > 16384) grouping, runs longer than 64 members (Zipf), I32 and I64 ids, an empty batch.  Rows no id
  touched keep their bits."""
  kw = _RULES[rule]
  id_dtype = np.int32 if (n + d + len(rule)) % 2 else np.int64
  rng = np.random.RandomState(n + d + len(rule))
  rows = _rows(d)
  x, a, z = _state(rng, (rows, d))
  x0, a0, z0 = x.copy(), a.copy(), z.copy()
  tx, ta, tz = cu(x), cu(a), cu(z)
  touched = np.zeros(rows, bool)
  zeros = 0
  for t in range(1, 4):
    ids = _ids(rng, n, rows, kind)
    g = (rng.normal(size=(n, d)) * 0.01).astype(np.float32)
    ops.sparse_ftrl_(tx, ta, tz, cu(ids.astype(id_dtype)), cu(g), **_op_rule(ops, kw))
    x, a, z = fo.ftrl_sparse(x, a, z, ids, g, **kw)
    for name, got, want in (("table", tx, x), ("accum", ta, a), ("linear", tz, z)):
      np.testing.assert_array_equal(bits(host(got)), bits(want), err_msg=f"{name} after step {t}")
    ok = ids[(ids >= 0) & (ids < rows)]
    touched[ok] = True
    zeros += int((bits(x[ok]) == 0).sum())
  for got, was in ((tx, x0), (ta, a0), (tz, z0)):
    assert np.array_equal(bits(host(got)[~touched]), bits(was[~touched]))
  if n > 1:
    assert zeros > 0, "l1 > 0 should have set some weights to exactly zero"


def test_sparse_ftrl_id_dtypes_agree(ops):
  """The same batch as I32 and as I64 ids gives the same bits; planted -1 and `rows` are skipped."""
  rng = np.random.RandomState(7)
  rows, d = 1001, 16
  x, a, z = _state(rng, (rows, d))
  ids = np.array([0, 5, 5, -1, rows, rows - 1, 5, 900], np.int64)
  g = rng.normal(size=(ids.size, d)).astype(np.float32)
  kw = _RULES["sqrt_shrink_beta"]
  want = fo.ftrl_sparse(x, a, z, ids, g, **kw)
  for id_dtype in (np.int32, np.int64):
    tx, ta, tz = cu(x), cu(a), cu(z)
    ops.sparse_ftrl_(tx, ta, tz, cu(ids.astype(id_dtype)), cu(g), **_op_rule(ops, kw))
    for got, exp in zip((tx, ta, tz), want):
      np.testing.assert_array_equal(bits(host(got)), bits(exp))


def test_sparse_ftrl_deterministic(ops):
  """Two identical Zipf runs give identical bits (both groupings, both power modes)."""
  for n, rule in ((16384, "sqrt"), (100_000, "sqrt_shrink_beta"), (100_000, "const")):
    rng = np.random.RandomState(11)
    rows, d = 20_000, 64
    x, a, z = _state(rng, (rows, d))
    ids = cu(_ids(rng, n, rows, "zipf")); g = cu((rng.normal(size=(n, d)) * 0.01).astype(np.float32))
    outs = []
    for _ in range(2):
      tx, ta, tz = cu(x), cu(a), cu(z)
      for _ in range(2):
        ops.sparse_ftrl_(tx, ta, tz, ids, g, **_op_rule(ops, _RULES[rule]))
      outs.append([bits(host(s)) for s in (tx, ta, tz)])
    for p, q in zip(*outs):
      assert np.array_equal(p, q)


# ------------------------------------------------------------------------------------------------
# the fp64-pow power mode: P differs from the oracle's by at most one fp32 ulp
# ------------------------------------------------------------------------------------------------
U = 2.0 ** -23   # one fp32 ulp, relative


def _bars(x, a, z, g, kw):
  """Bars on |lin' - lin'_oracle| and |var' - var'_oracle| for one step from the state (x, a, z), when each P(.) may be one
  fp32 ulp off the oracle's (DESIGN.md section 2, A17).  Every later fp32 operation adds at most one ulp of its result;
  the factor 2 covers the second-order terms and the float64 evaluation of the bar itself."""
  x, a, z, g = (np.asarray(t, np.float64) for t in (x, a, z, g))
  lr = float(np.float32(kw["lr"]))
  s = float(np.float32(kw.get("l2_shrinkage", 0.0)))
  l2a = float(fo.l2a(kw["l2"], kw.get("beta", 0.0), kw["lr"]))
  p = -float(np.float32(kw["lr_power"]))
  na = a + g * g
  pn, pa = na ** p, a ** p
  sigma = (pn - pa) / lr
  gs = g + 2 * s * x if s > 0 else g
  lin1 = z + (gs - sigma * x)
  bar_lin = 2 * U * (np.abs(x) * (pn + pa + np.abs(pn - pa)) / lr + 2 * np.abs(sigma * x) + np.abs(gs - sigma * x)
                     + np.abs(lin1))
  y = pn / lr + 2 * l2a
  var1 = np.where(np.abs(lin1) > kw["l1"], (np.sign(lin1) * kw["l1"] - lin1) / y, 0.0)
  bar_var = 2 * (bar_lin / y + 5 * U * np.abs(var1))
  return bar_lin, bar_var


def _check_pow_step(got, want, bars, what, stats):
  (gx, ga, gz), (wx, wa, wz), (bl, bv) = got, want, bars
  np.testing.assert_array_equal(bits(ga), bits(wa), err_msg=f"accum, {what}")
  assert (np.abs(gz.astype(np.float64) - wz) <= bl).all(), f"linear outside the bar, {what}"
  assert (np.abs(gx.astype(np.float64) - wx) <= bv).all(), f"var outside the bar, {what}"
  stats[0] += int((bits(gx) != bits(wx)).sum() + (bits(gz) != bits(wz)).sum())
  stats[1] += 2 * wx.size


@pytest.mark.parametrize("lr_power", [-0.3, -0.75])
@pytest.mark.parametrize("shrink_beta", [False, True])
def test_pow_mode_inside_the_ulp_bar(ops, lr_power, shrink_beta):
  """lr_power other than -0.5 and 0: each step starts from the oracle's state.  accum is bit-exact; linear and var lie
  inside the bar, and at most 1e-5 of the elements differ in any bit."""
  kw = dict(lr=0.05, lr_power=lr_power, l1=0.02, l2=0.01)
  if shrink_beta:
    kw.update(l2_shrinkage=0.3, beta=0.5)
  rng = np.random.RandomState(17 + int(shrink_beta))
  stats = [0, 0]
  # sparse: Zipf ids (long runs) on a 20k x 64 table
  rows, d, n = 20_000, 64, 16384
  x, a, z = _state(rng, (rows, d))
  for t in range(3):
    ids = _ids(rng, n, rows, "zipf")
    g = (rng.normal(size=(n, d)) * 0.01).astype(np.float32)
    tx, ta, tz = cu(x), cu(a), cu(z)
    ops.sparse_ftrl_(tx, ta, tz, cu(ids), cu(g), **_op_rule(ops, kw))
    heads, gsum = fo._summed_rows(ids, g, rows)
    want = fo.ftrl_sparse(x, a, z, ids, g, **kw)
    got = [host(s) for s in (tx, ta, tz)]
    others = np.setdiff1d(np.arange(rows), heads)
    for s, was in zip(got, (x, a, z)):
      assert np.array_equal(bits(s[others]), bits(was[others]))
    _check_pow_step([s[heads] for s in got], [s[heads] for s in want],
                    _bars(x[heads], a[heads], z[heads], gsum, kw), f"sparse step {t}", stats)
    x, a, z = want
  # dense: 40 variables, two steps
  sizes = [int(s) for s in rng.randint(1, 5000, size=40)]
  xs = [_state(rng, (s,)) for s in sizes]
  for t in range(2):
    gs = [(rng.normal(size=s) * 0.05).astype(np.float32) for s in sizes]
    tv = [[cu(c) for c in st] for st in xs]
    ops.ftrl_dense_([v[0] for v in tv], [cu(g) for g in gs], [v[1] for v in tv], [v[2] for v in tv],
                    **_op_rule(ops, kw))
    for i in range(len(sizes)):
      want = fo.ftrl_dense(*xs[i], gs[i], **kw)
      _check_pow_step([host(c) for c in tv[i]], want, _bars(*xs[i], gs[i], kw), f"variable {i}, dense step {t}", stats)
      xs[i] = want
  assert stats[0] <= 1e-5 * stats[1], stats


# ------------------------------------------------------------------------------------------------
# dense multi-tensor kernel
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("rule", ["sqrt_shrink_beta", "const"])
def test_dense_ftrl_bit_exact_many_variables(ops, rule):
  """1006 variables: more than one launch's parameters hold (736), so two launches; numels 0, 1, 1023, 1025 and about
  3M."""
  kw = _RULES[rule]
  rng = np.random.RandomState(3)
  sizes = [(0,), (1,), (1023,), (1025,), (3_000_017,), (845, 512)] + [(int(s),) for s in rng.randint(1, 40, size=998)]
  sizes += [(0,), (7, 5)]
  assert len(sizes) == 1006
  st = [_state(rng, s) for s in sizes]
  tv = [[cu(c) for c in s] for s in st]
  for t in (1, 2):
    gs = [(rng.normal(size=s) * 0.05).astype(np.float32) for s in sizes]
    ops.ftrl_dense_([v[0] for v in tv], [cu(g) for g in gs], [v[1] for v in tv], [v[2] for v in tv], **_op_rule(ops, kw))
    for i in range(len(sizes)):
      st[i] = fo.ftrl_dense(*st[i], gs[i], **kw)
      for name, got, want in zip(("var", "accum", "linear"), tv[i], st[i]):
        np.testing.assert_array_equal(bits(host(got)), bits(want), err_msg=f"{name} of variable {i}, step {t}")


# ------------------------------------------------------------------------------------------------
# errors
# ------------------------------------------------------------------------------------------------
def test_ftrl_argument_errors(ops):
  t = torch.zeros((10, 4), device="cuda"); a = torch.full_like(t, 0.1); z = torch.zeros_like(t)
  ids = torch.zeros((2,), dtype=torch.int64, device="cuda"); g = torch.ones((2, 4), device="cuda")
  rule = dict(lr=0.1, lr_power=-0.5, l1=0.0, l2a=0.0, l2_shrinkage=0.0)
  with pytest.raises(RuntimeError, match="CUDA"):
    ops.sparse_ftrl_(t.cpu(), a, z, ids, g, **rule)
  with pytest.raises(RuntimeError, match="CUDA"):
    ops.sparse_ftrl_(t, a, z, ids.cpu(), g, **rule)
  with pytest.raises(RuntimeError, match="CUDA"):
    ops.ftrl_dense_([t.cpu()], [g.cpu()], [a.cpu()], [z.cpu()], **rule)
  with pytest.raises(ValueError, match="grad_rows"):
    ops.sparse_ftrl_(t, a, z, ids, g[:1], **rule)
  with pytest.raises(ValueError, match="accum must be"):
    ops.sparse_ftrl_(t, a[:5], z, ids, g, **rule)
  with pytest.raises(ValueError, match="linear must be"):
    ops.sparse_ftrl_(t, a, torch.zeros((10, 5), device="cuda"), ids, g, **rule)
  with pytest.raises(ValueError, match="same length"):
    ops.ftrl_dense_([t], [g], [a], [], **rule)
  with pytest.raises(ValueError, match="shape"):
    ops.ftrl_dense_([t], [t], [a[:3]], [z], **rule)
  with pytest.raises(ValueError, match="contiguous"):
    ops.ftrl_dense_([t], [t], [a], [z.t()], **rule)
  # scalars, checked by the library and reported across the ABI, on both entry points
  bad = [dict(lr=0.0), dict(lr=-0.1), dict(lr=float("nan")), dict(lr=float("inf")), dict(lr_power=0.5),
         dict(lr_power=float("nan")), dict(l1=-1e-3), dict(l1=float("inf")), dict(l2a=-1e-3), dict(l2a=float("nan")),
         dict(l2_shrinkage=-1e-3), dict(l2_shrinkage=float("-inf"))]
  for b in bad:
    with pytest.raises(ValueError, match="sparse_ftrl"):
      ops.sparse_ftrl_(t, a, z, ids, g, **dict(rule, **b))
    with pytest.raises(ValueError, match="ftrl_dense"):
      ops.ftrl_dense_([t], [t], [a], [z], **dict(rule, **b))
  # limits checked by the library
  wide = torch.zeros((3, 1025), device="cuda")
  with pytest.raises(ValueError, match="d=1025"):
    ops.sparse_ftrl_(wide, torch.zeros_like(wide), torch.zeros_like(wide), ids, torch.zeros((2, 1025), device="cuda"),
                     **rule)
  n = 1 << 24
  t1 = torch.zeros((4, 1), device="cuda")
  with pytest.raises(ValueError, match="2\\^24"):
    ops.sparse_ftrl_(t1, torch.zeros_like(t1), torch.zeros_like(t1), torch.zeros((n,), dtype=torch.int32, device="cuda"),
                     torch.ones((n, 1), device="cuda"), **rule)
  # nothing was written by any refused call
  torch.cuda.synchronize()
  assert torch.count_nonzero(t) == 0 and torch.count_nonzero(z) == 0 and bool((a == 0.1).all())
  assert torch.count_nonzero(t1) == 0


# ------------------------------------------------------------------------------------------------
# the optimizer class, end to end
# ------------------------------------------------------------------------------------------------
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


def test_composite_optimizer_with_ftrl_matches_its_parts(tfrs):
  """composite_optimizer_test.py:28-86 for the (Ftrl: tables, Adagrad: dense) pair, 10 steps."""
  torch.manual_seed(0)
  CompositeOptimizer = tfrs.experimental.optimizers.CompositeOptimizer
  a = _Tiny(tfrs); b = _copy(tfrs, a)
  make = lambda: tfrs.optimizers.Ftrl(0.05, l1_regularization_strength=1e-3, l2_regularization_strength=1e-2,
                                      l2_shrinkage_regularization_strength=0.1, beta=0.2)
  c1, c2 = make(), tfrs.optimizers.Adagrad(0.1)
  comp = CompositeOptimizer([(c1, lambda: [a.emb1, a.emb2._anchor]), (c2, lambda: [a.w, a.b])]).bind(a)
  s1, s2 = make(), tfrs.optimizers.Adagrad(0.1)
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
  # the composite's Ftrl state equals the standalone optimizer's
  for p, q in zip(c1.variables(), s1.variables()):
    assert torch.equal(p.view(torch.int32), q.view(torch.int32))


def test_tpu_embedding_model_first_step_equals_the_oracle(tfrs):
  """A TPUEmbedding model under `Model.compile`: after one step, each table equals the oracle's sparse rule on the
  (ids, rows) pair it received and each dense parameter the dense rule on its gradient, bit for bit; rows no id touched
  keep their bits."""
  torch.manual_seed(0)
  E = tfrs.layers.embedding
  t_video, t_user = E.TableConfig(500, 8, combiner="mean"), E.TableConfig(300, 4, combiner="sum")
  fcs = {"watched": E.FeatureConfig(t_video), "favorited": E.FeatureConfig(t_video), "friends": E.FeatureConfig(t_user)}

  class M(tfrs.Model):

    def __init__(self):
      super().__init__()
      self.embedding = E.TPUEmbedding(fcs)
      self.top = tfrs.layers.blocks.MLP([16, 1])

    def compute_loss(self, inputs, training=False):
      feats, labels = inputs
      acts = self.embedding(feats)
      pred = self.top(torch.cat([acts[k] for k in sorted(acts)], -1))
      return ((pred.view(-1) - labels) ** 2).mean()

  rng = np.random.RandomState(1)
  B = 64
  feats = {}
  for name, vocab in (("watched", 500), ("favorited", 500), ("friends", 300)):
    lens = rng.randint(0, 6, size=B)
    sp = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    feats[name] = (cu(rng.randint(0, vocab, size=int(sp[-1])).astype(np.int32)), sp)
  labels = cu(rng.rand(B).astype(np.float32))
  model = M()
  opt = tfrs.optimizers.Ftrl(0.1, l1_regularization_strength=1e-3, l2_regularization_strength=1e-3,
                             l2_shrinkage_regularization_strength=0.05, beta=0.1)
  model.compile(optimizer=opt)
  opt.zero_grad()
  model.compute_loss((feats, labels), training=True).backward()
  tables = model.embedding._tables
  before = [host(t.weight).copy() for t in tables]
  pairs = [[(host(i).reshape(-1), host(g)) for i, g in t._sparse_grads] for t in tables]
  dense = tfrs.optimizers.dense_variables(model)
  dense_before = [(host(p).copy(), host(p.grad).copy()) for p in dense]
  assert len(dense) == 4 and all(len(p) == 1 for p in pairs)
  opt.apply_gradients()
  kw = dict(lr=0.1, l1=1e-3, l2=1e-3, l2_shrinkage=0.05, beta=0.1)
  for t, w, ((ids, rows),) in zip(tables, before, pairs):
    init = np.full_like(w, 0.1)
    want = fo.ftrl_sparse(w, init, np.zeros_like(w), ids, rows, **kw)
    for got, exp in zip((t.weight, t._tfrs_ftrl_acc, t._tfrs_ftrl_linear), want):
      np.testing.assert_array_equal(bits(host(got)), bits(exp))
    untouched = np.setdiff1d(np.arange(w.shape[0]), ids)
    assert np.array_equal(bits(host(t.weight)[untouched]), bits(w[untouched]))
  for p, (w, g) in zip(dense, dense_before):
    want = fo.ftrl_dense(w, np.full_like(w, 0.1), np.zeros_like(w), g, **kw)
    for got, exp in zip((p, p._tfrs_ftrl_acc, p._tfrs_ftrl_linear), want):
      np.testing.assert_array_equal(bits(host(got)), bits(exp))
  losses = [float(model.train_step((feats, labels))["loss"]) for _ in range(20)]
  assert np.isfinite(losses).all() and losses[-1] < losses[0], losses
  assert opt.iterations == 21 and len(opt.variables()) == 2 * (2 + 4)


def _synthetic_data(num_dense, vocab_sizes, dataset_size, batch_size, seed=0):
  """experimental/models/ranking_test.py:_generate_synthetic_data: labels = int((mean(dense) + sum(ids)/sum(vocab)) / 2 + 0.5)."""
  g = torch.Generator(device="cuda"); g.manual_seed(seed)
  dense = torch.rand((dataset_size, num_dense), generator=g, device="cuda")
  sparse = [torch.randint(0, v, (dataset_size,), generator=g, device="cuda", dtype=torch.int32) for v in vocab_sizes]
  labels = ((dense.mean(1) + torch.stack(sparse, -1).sum(1).float() / sum(vocab_sizes)) / 2.0 + 0.5).to(torch.int32)
  return [({"dense_features": dense[lo:lo + batch_size],
            "sparse_features": {str(i): s[lo:lo + batch_size] for i, s in enumerate(sparse)}}, labels[lo:lo + batch_size])
          for lo in range(0, dataset_size - batch_size + 1, batch_size)]


def test_ranking_model_trains_with_ftrl(tfrs):
  """ranking_test.py's Ranking model compiled with Ftrl(0.1) lowers its loss."""
  vocab = [30, 3, 26]
  torch.manual_seed(1)
  model = tfrs.experimental.models.Ranking(
      embedding_layer=torch.nn.ModuleDict({str(i): tfrs.layers.embedding.Embedding(v, 16) for i, v in enumerate(vocab)}),
      feature_interaction=tfrs.layers.feature_interaction.DotInteraction())
  model.compile(optimizer=tfrs.optimizers.Ftrl(0.1))
  data = _synthetic_data(8, vocab, 64, 16, seed=5)
  losses = [float(model.evaluate(data)["loss"])]
  for _ in range(15):
    model.fit(data, epochs=1)
    losses.append(float(model.evaluate(data)["loss"]))
  assert np.isfinite(losses).all() and losses[-1] < losses[0], losses
  assert model.optimizer.iterations == 15 * len(data)
  for p in model.parameters():
    assert torch.isfinite(p).all()


def test_unified_embedding_model_first_step_equals_the_oracle(tfrs):
  """Several features share each UnifiedEmbedding table, so a table's gradient rows in a step come from several features'
  values; the first step equals the oracle on them, and training goes on without error."""
  from recommenders_b200.layers.feature_multiplexing import unified_embedding as ue_mod
  torch.manual_seed(0)
  names = ["movie_id", "user_id", "user_gender"]
  cfg = ue_mod.UnifiedEmbeddingConfig(buckets_per_table=500, dim_per_table=8, num_tables=2, name="unified_table")
  for n in names:
    cfg.add_feature(n, 2)
  ue = ue_mod.UnifiedEmbedding(cfg, None)

  class UnifiedEmbeddingModel(tfrs.models.Model):
    def __init__(self):
      super().__init__()
      self.embedding = ue
      self.network = tfrs.layers.blocks.MLP([32, 1], final_activation="sigmoid")
      self.task = tfrs.tasks.Ranking()

    def compute_loss(self, inputs, training=False):
      feats, labels = inputs
      return self.task(labels, self.network(torch.cat(self.embedding(feats), -1)))

  rng = np.random.default_rng(5)
  data = []
  for _ in range(10):
    uid, mid = rng.integers(0, 200, size=256), rng.integers(0, 300, size=256)
    feats = {"movie_id": np.char.mod("%d", mid), "user_id": np.char.mod("%d", uid),
             "user_gender": np.where(uid % 2 == 0, "True", "False")}
    data.append((feats, torch.from_numpy(((uid + mid) % 3 == 0).astype(np.float32)).cuda().reshape(-1, 1)))
  opt = tfrs.optimizers.Ftrl(0.05, l1_regularization_strength=1e-4)
  model = UnifiedEmbeddingModel()
  model.compile(optimizer=opt)
  opt.zero_grad()
  model.compute_loss(data[0], training=True).backward()
  before = [host(t.weight) for t in ue._tables]
  pairs = [[(host(i).reshape(-1), host(g)) for i, g in t._sparse_grads] for t in ue._tables]
  assert all(sum(i.size for i, _ in p) > 256 for p in pairs)
  opt.apply_gradients()
  for t, w, p in zip(ue._tables, before, pairs):
    ids = np.concatenate([i for i, _ in p]); g = np.concatenate([r.reshape(-1, w.shape[1]) for _, r in p])
    want = fo.ftrl_sparse(w, np.full_like(w, 0.1), np.zeros_like(w), ids, g, lr=0.05, l1=1e-4)
    for got, exp in zip((t.weight, t._tfrs_ftrl_acc, t._tfrs_ftrl_linear), want):
      np.testing.assert_array_equal(bits(host(got)), bits(exp))
  losses = [float(model.train_step(b)["loss"]) for b in data]
  assert np.isfinite(losses).all()
  assert all(t._sparse_grads == [] for t in ue._tables)
  assert opt.iterations == 11
