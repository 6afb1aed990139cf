"""GPU tests of K7 (ClippyAdagrad, csrc/clippy_adagrad.cu) and of experimental.optimizers: the sparse and the dense
multi-tensor kernels bit-exact against the fp32 restatement in tests/clippy_oracle.py, the reference's step tests through the public class
(experimental/optimizers/clippy_adagrad_test.py:164-303), CompositeOptimizer against its parts
(composite_optimizer_test.py:28-86), and end-to-end training.  Run with -m gpu."""
import itertools
import os
import sys

import numpy as np
import pytest
import torch

from oracle import oracle as orc

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import clippy_oracle as co  # noqa: E402

pytestmark = pytest.mark.gpu


def cu(a):
  return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def bits(a):
  return np.ascontiguousarray(a, np.float32).view(np.uint32)


@pytest.fixture(scope="module")
def tfrs():
  import recommenders_b200 as t
  return t


def _ids(rng, n, rows, kind):
  ids = np.minimum(rng.zipf(1.05, size=n) - 1, rows - 1) if kind == "zipf" else rng.randint(0, rows, size=n)
  ids = ids.astype(np.int64)
  if n > 1:
    ids[::97] = -1          # out-of-range ids are skipped
    ids[5::101] = rows
  return ids


def _sparse_case(n, d, kind, seed):
  rng = np.random.RandomState(seed)
  rows = max(64, min(100_000, 2_000_000 // d))
  ids = _ids(rng, n, rows, kind)
  table = rng.uniform(-0.05, 0.05, size=(rows, d)).astype(np.float32)
  acc = rng.uniform(0.05, 0.2, size=(rows, d)).astype(np.float32)
  g = (rng.normal(size=(n, d)) * 0.01).astype(np.float32)
  return ids, table, acc, g


def _run_sparse(ops, ids, table, acc, g, id_dtype=np.int64, **kw):
  tt, ta = cu(table), cu(acc)
  f = torch.zeros((), device="cuda")
  ops.sparse_clippy_adagrad_(tt, ta, cu(ids.astype(id_dtype)), cu(g), clipping_factor=f, **kw)
  return tt.cpu().numpy(), ta.cpu().numpy(), f.cpu().numpy()


def _rule(lr=0.5, eps=1e-7, var_rel=0.1, acc_rel=0.0, abs_thr=1e-7, flags=0):
  ours = dict(lr=lr, eps=eps, variable_relative_threshold=var_rel, accumulator_relative_threshold=acc_rel,
              absolute_threshold=abs_thr, clip_accumulator_update=bool(flags & 1),
              use_standard_accumulator_update=bool(flags & 2))
  ref = dict(lr=lr, eps=eps, var_rel=var_rel, acc_rel=acc_rel, abs_thr=abs_thr, clip_accumulator_update=bool(flags & 1),
             use_standard_accumulator_update=bool(flags & 2))
  return ours, ref


def _assert_sparse_bit_exact(ops, ids, table, acc, g, id_dtype=np.int64, **rule):
  ours, ref = _rule(**rule)
  et, ea, ef = co.clippy_adagrad_sparse(table, acc, ids, g, **ref)
  t, a, f = _run_sparse(ops, ids, table, acc, g, id_dtype, **ours)
  np.testing.assert_array_equal(bits(f), bits(ef))
  np.testing.assert_array_equal(bits(t), bits(et))
  np.testing.assert_array_equal(bits(a), bits(ea))
  return ef


# ------------------------------------------------------------------------------------------------
# sparse kernel
# ------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def ops():
  from recommenders_b200 import ops as o
  return o


_SPARSE = [(n, kind, d) for n in (1, 100, 16384, 20000) for kind in ("uniform", "zipf") for d in (1, 3, 64, 128, 1024)]


@pytest.mark.parametrize("n,kind,d", _SPARSE)
def test_sparse_clippy_adagrad_bit_exact(ops, n, kind, d):
  """Both grouping paths (rank sort n <= 16384, bitonic above), runs longer than 64 (Zipf), I32 and I64 ids."""
  ids, table, acc, g = _sparse_case(n, d, kind, seed=n + d)
  id_dtype = np.int32 if (n + d) % 2 else np.int64
  f = _assert_sparse_bit_exact(ops, ids, table, acc, g, id_dtype, lr=0.5, var_rel=0.1, acc_rel=1e-3, abs_thr=1e-4)
  assert 0.0 < f <= 1.0


@pytest.mark.parametrize("flags,acc_rel", list(itertools.product((0, 1, 2), (0.0, 1e-3))))
@pytest.mark.parametrize("id_dtype", [np.int32, np.int64])
def test_sparse_clippy_adagrad_flags(ops, flags, acc_rel, id_dtype):
  ids, table, acc, g = _sparse_case(3000, 32, "zipf", seed=11 + flags)
  f = _assert_sparse_bit_exact(ops, ids, table, acc, g, id_dtype, lr=0.3, var_rel=0.2, acc_rel=acc_rel, abs_thr=1e-6,
                               flags=flags)
  assert f < 1.0   # the clip is active on this batch
  # no clipping: the plain Adagrad-like step, factor exactly 1
  f = _assert_sparse_bit_exact(ops, ids, table, acc, g, id_dtype, lr=1e-4, var_rel=0.1, acc_rel=acc_rel, abs_thr=1.0,
                               flags=flags)
  assert f == 1.0


@pytest.mark.parametrize("flags", [0, 1, 2])
def test_sparse_clippy_adagrad_zero_factor(ops, flags):
  """abs_thr = 0 and a zero reference element: factor 0, no variable update, the accumulator still per the rule."""
  ids, table, acc, g = _sparse_case(500, 16, "uniform", seed=5)
  table[ids[10]] = 0.0
  f = _assert_sparse_bit_exact(ops, ids, table, acc, g, lr=0.5, var_rel=0.1, abs_thr=0.0, flags=flags)
  assert f == 0.0
  t, a, _ = _run_sparse(ops, ids, table, acc, g, **_rule(lr=0.5, var_rel=0.1, abs_thr=0.0, flags=flags)[0])
  assert np.array_equal(t, table)
  touched = np.unique(ids[(ids >= 0) & (ids < table.shape[0])])
  if flags == 1:
    assert np.array_equal(a, acc)             # clipped accumulator update: u = g * 0
  else:
    assert (a[touched] > acc[touched]).any()  # a + g*g


def test_sparse_clippy_adagrad_reproducible_and_empty(ops):
  ids, table, acc, g = _sparse_case(20000, 64, "zipf", seed=3)
  rule = _rule(var_rel=0.1, acc_rel=1e-3)[0]
  r1 = _run_sparse(ops, ids, table, acc, g, **rule)
  r2 = _run_sparse(ops, ids, table, acc, g, **rule)
  for x, y in zip(r1, r2):
    np.testing.assert_array_equal(bits(x), bits(y))
  # nothing touched (empty batch, or only out-of-range ids): state unchanged, factor 1
  for bad in (np.zeros((0,), np.int64), np.array([-1, table.shape[0]], np.int64)):
    t, a, f = _run_sparse(ops, bad, table, acc, np.ones((bad.size, 64), np.float32), **rule)
    assert np.array_equal(bits(t), bits(table)) and np.array_equal(bits(a), bits(acc)) and f == 1.0


def test_sparse_clippy_adagrad_argument_errors(ops):
  t = torch.zeros((10, 4), device="cuda"); a = torch.zeros_like(t)
  ids = torch.zeros((2,), dtype=torch.int64, device="cuda"); g = torch.zeros((2, 4), device="cuda")
  rule = _rule()[0]
  with pytest.raises(ValueError, match="non-negative"):
    ops.sparse_clippy_adagrad_(t, a, ids, g, **dict(rule, variable_relative_threshold=-0.1))
  with pytest.raises(ValueError, match="not both"):
    ops.sparse_clippy_adagrad_(t, a, ids, g, **dict(rule, clip_accumulator_update=True, use_standard_accumulator_update=True))
  with pytest.raises(ValueError, match="grad_rows"):
    ops.sparse_clippy_adagrad_(t, a, ids, g[:1], **rule)


# ------------------------------------------------------------------------------------------------
# dense multi-tensor kernel
# ------------------------------------------------------------------------------------------------
def _dense_case(sizes, seed):
  rng = np.random.RandomState(seed)
  vs = [rng.uniform(-0.5, 0.5, size=s).astype(np.float32) for s in sizes]
  accs = [rng.uniform(0.05, 0.2, size=s).astype(np.float32) for s in sizes]
  gs = [(rng.normal(size=s) * 0.05).astype(np.float32) for s in sizes]
  return vs, accs, gs


def _assert_dense_bit_exact(ops, sizes, seed, **rule):
  ours, ref = _rule(**rule)
  vs, accs, gs = _dense_case(sizes, seed)
  tv = [cu(v) for v in vs]; ta = [cu(a) for a in accs]
  f = torch.full((len(sizes),), -1.0, device="cuda")
  ops.clippy_adagrad_dense_(tv, [cu(g) for g in gs], ta, clipping_factors=f, **ours)
  fs = f.cpu().numpy()
  for i in range(len(sizes)):
    ev, ea, ef = co.clippy_adagrad_dense(vs[i], accs[i], gs[i], **ref)
    np.testing.assert_array_equal(bits(fs[i]), bits(ef), err_msg=f"variable {i}")
    np.testing.assert_array_equal(bits(tv[i].cpu().numpy()), bits(ev), err_msg=f"variable {i}")
    np.testing.assert_array_equal(bits(ta[i].cpu().numpy()), bits(ea), err_msg=f"variable {i}")
  return fs


@pytest.mark.parametrize("flags,acc_rel", [(0, 0.0), (1, 1e-3), (2, 0.0), (2, 1e-3)])
def test_dense_clippy_adagrad_bit_exact(ops, flags, acc_rel):
  sizes = [(1,), (3,), (1000,), (845, 512), (0,), (7, 5), (512,), (1025,), (256, 1)]
  fs = _assert_dense_bit_exact(ops, sizes, seed=flags, lr=0.3, var_rel=0.1, acc_rel=acc_rel, abs_thr=1e-4, flags=flags)
  assert fs[4] == 1.0 and (fs < 1.0).any()


def test_dense_clippy_adagrad_many_variables(ops):
  """More variables than one launch's parameters hold (896 per launch): several batches, one factor per variable."""
  rng = np.random.RandomState(1)
  sizes = [(int(s),) for s in rng.randint(1, 40, size=2000)]
  _assert_dense_bit_exact(ops, sizes, seed=2, lr=0.3, var_rel=0.1, abs_thr=1e-4)


def test_dense_clippy_adagrad_zero_factor(ops):
  vs, accs, gs = _dense_case([(33,)], seed=4)
  vs[0][7] = 0.0
  ours, ref = _rule(var_rel=0.1, abs_thr=0.0)
  tv, ta = cu(vs[0]), cu(accs[0])
  f = torch.zeros((1,), device="cuda")
  ops.clippy_adagrad_dense_([tv], [cu(gs[0])], [ta], clipping_factors=f, **ours)
  ev, ea, ef = co.clippy_adagrad_dense(vs[0], accs[0], gs[0], **ref)
  assert ef == 0.0 and float(f[0]) == 0.0 and np.array_equal(tv.cpu().numpy(), vs[0])
  np.testing.assert_array_equal(bits(ta.cpu().numpy()), bits(ea))


# ------------------------------------------------------------------------------------------------
# ClippyAdagradTest (clippy_adagrad_test.py:164-303) through the public class, float32 state
# ------------------------------------------------------------------------------------------------
F32_TOL = dict(rtol=1e-6, atol=1e-6)


def _reference_step(tfrs, dense_g, sparse_g, **kw):
  m = torch.nn.Module()
  m.x = torch.nn.Parameter(torch.tensor([1.0, 2.0], device="cuda"))
  m.sparse_x = tfrs.layers.embedding.Embedding(2, 2)
  m.sparse_x.weight.copy_(torch.tensor([[3.0, 4.0], [1.0, 2.0]]))
  opt = tfrs.experimental.optimizers.ClippyAdagrad(export_clipping_factors=True, **kw).bind(m)
  opt.zero_grad()
  m.x.grad = torch.tensor(dense_g, device="cuda")
  m.sparse_x._sparse_grads.append((torch.tensor([1], device="cuda"), torch.tensor([sparse_g], device="cuda")))
  opt.apply_gradients()
  assert opt.iterations == 1
  factors = [float(f) for f in opt.clipping_factors]   # [sparse_x, x]: tables first
  return (m.x.detach().cpu().numpy(), m.sparse_x.weight.cpu().numpy(), m.x._tfrs_clippy_acc.cpu().numpy(),
          m.sparse_x._tfrs_clippy_acc.cpu().numpy(), factors)


def test_step_no_clip(tfrs):
  lr, s0 = 0.1, 0.1
  x, sx, xa, sa, f = _reference_step(tfrs, [0.1, 0.15], [0.1, 0.15], learning_rate=lr, initial_accumulator_value=s0 ** 2)
  np.testing.assert_allclose(x, [1.0 - lr * 0.1 / s0, 2.0 - lr * 0.15 / s0], **F32_TOL)
  np.testing.assert_allclose(sx, [[3.0, 4.0], [1.0 - lr * 0.1 / s0, 2.0 - lr * 0.15 / s0]], **F32_TOL)
  np.testing.assert_allclose(xa, [s0 ** 2 + 0.1 ** 2, s0 ** 2 + 0.15 ** 2], **F32_TOL)
  np.testing.assert_allclose(sa, [[s0 ** 2, s0 ** 2], [s0 ** 2 + 0.1 ** 2, s0 ** 2 + 0.15 ** 2]], **F32_TOL)
  np.testing.assert_allclose(f, [1.0, 1.0], **F32_TOL)


@pytest.mark.parametrize("clip_accumulator_update", [False, True])
def test_step_clip(tfrs, clip_accumulator_update):
  lr, s0 = 0.2, 0.1
  x, sx, xa, sa, f = _reference_step(tfrs, [10.0, 10.0], [10.0, 10.0], learning_rate=lr, initial_accumulator_value=s0 ** 2,
                                     variable_relative_threshold=0.4, accumulator_relative_threshold=0.01,
                                     absolute_threshold=0.1, epsilon=0.0, clip_accumulator_update=clip_accumulator_update)
  np.testing.assert_allclose(x, [0.4, 1.4], **F32_TOL)
  np.testing.assert_allclose(sx, [[3.0, 4.0], [0.4, 1.4]], **F32_TOL)
  factor = 0.6 * s0 / (10.0 * lr)
  np.testing.assert_allclose(f, [factor, factor], **F32_TOL)
  u = (f[1] * 10, f[0] * 10) if clip_accumulator_update else (10.0, 10.0)
  np.testing.assert_allclose(xa, [s0 ** 2 + u[0] ** 2] * 2, **F32_TOL)
  np.testing.assert_allclose(sa, [[s0 ** 2, s0 ** 2], [s0 ** 2 + u[1] ** 2] * 2], **F32_TOL)


def test_step_standard_update(tfrs):
  lr = 0.1
  x, sx, xa, sa, f = _reference_step(tfrs, [0.1, 0.15], [0.1, 0.15], learning_rate=lr, initial_accumulator_value=0.0,
                                     use_standard_accumulator_update=True)
  np.testing.assert_allclose(x, [1.0 - lr, 2.0 - lr], **F32_TOL)
  np.testing.assert_allclose(sx, [[3.0, 4.0], [1.0 - lr, 2.0 - lr]], **F32_TOL)
  np.testing.assert_allclose(xa, np.square(np.float32([0.1, 0.15])), **F32_TOL)
  np.testing.assert_allclose(sa, [[0.0, 0.0], [0.1 ** 2, 0.15 ** 2]], **F32_TOL)
  np.testing.assert_allclose(f, [1.0, 1.0], **F32_TOL)


def test_shrink_by_references_on_cuda(tfrs):
  """ClipByReferenceTest (clippy_adagrad_test.py:21-160) on the product's helper, against the float64 oracle."""
  shrink = tfrs.experimental.optimizers.shrink_by_references
  cases = [(2., [4.], [0.1], 0.02), (-2., [4.], [0.1], 0.), (-2., [0.], [0.1], 0.), (2., [20.], [0.1], 0.1),
           (0., [0.], [0.], 0.), (2., [4., -5.], [0.1, 0.2], 0.02), (2., [], [], 0.02),
           ([1., 1., 0., 0.], [[1., 0.1, 1., 0.]], [0.1], 0.), ([1., 1., 0., 0.], [[1., 0., 1., 0.]], [0.1], 0.),
           ([[1., 2.], [1., 2.]], [1.], [0.1], 0.1)]
  for tensor, refs, factors, absolute in cases:
    clipped, scale = shrink(torch.tensor(tensor, dtype=torch.float64, device="cuda"),
                            [torch.tensor(r, dtype=torch.float64, device="cuda") for r in refs], factors, absolute)
    ec, es = co.shrink_by_references(tensor, refs, factors, absolute)
    assert clipped.is_cuda and scale.is_cuda
    np.testing.assert_allclose(clipped.cpu().numpy(), ec, rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(float(scale), es, rtol=1e-12, atol=1e-12)
  clipped, scale = shrink(2., [4.], [0.1], 0.02)   # Python numbers go to the current device
  assert clipped.is_cuda and abs(float(scale) - 0.21) < 1e-6
  with pytest.raises(RuntimeError, match="CUDA"):
    shrink(torch.ones(2), [torch.ones(2)], [0.1], 0.1)


# ------------------------------------------------------------------------------------------------
# CompositeOptimizer (composite_optimizer_test.py:28-86)
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
  for a, b in ((dst.emb1.weight, src.emb1.weight), (dst.emb2.weight, src.emb2.weight)):
    a.copy_(b)
  with torch.no_grad():
    dst.w.copy_(src.w); dst.b.copy_(src.b)
  return dst


def _feed(model, step):
  g = torch.Generator(device="cuda"); g.manual_seed(step)
  for emb, n in ((model.emb1, 700), (model.emb2, 300)):
    ids = torch.randint(0, emb.input_dim, (n,), generator=g, device="cuda")
    rows = torch.randn((n, emb.output_dim), generator=g, device="cuda") * 0.1
    emb._sparse_grads += [(ids[:n // 2], rows[:n // 2]), (ids[n // 2:], rows[n // 2:])]   # two lookups of one table
  model.w.grad = torch.randn(model.w.shape, generator=g, device="cuda") * 0.1
  model.b.grad = torch.randn(model.b.shape, generator=g, device="cuda") * 0.1


def test_composite_optimizer_matches_its_parts(tfrs):
  torch.manual_seed(0)
  ClippyAdagrad, CompositeOptimizer = tfrs.experimental.optimizers.ClippyAdagrad, tfrs.experimental.optimizers.CompositeOptimizer
  a = _Tiny(tfrs); b = _copy(tfrs, a)
  kw = dict(learning_rate=0.2, variable_relative_threshold=0.2, accumulator_relative_threshold=1e-3,
            export_clipping_factors=True)
  c1, c2 = ClippyAdagrad(**kw), tfrs.optimizers.Adagrad(0.1)
  comp = CompositeOptimizer([(c1, lambda: [a.emb1, a.emb2._anchor]), (c2, lambda: [a.w, a.b])]).bind(a)
  assert comp.optimizers == [c1, c2]
  s1, s2 = ClippyAdagrad(**kw), tfrs.optimizers.Adagrad(0.1)
  for step in range(10):
    comp.zero_grad()
    _feed(a, step); _feed(b, step)
    comp.apply_gradients()
    s1.apply_gradients([b.emb1, b.emb2]); s2.apply_gradients([b.w, b.b])
    for x, y in ((a.emb1.weight, b.emb1.weight), (a.emb2.weight, b.emb2.weight), (a.w, b.w), (a.b, b.b)):
      assert torch.equal(x.detach().view(torch.int32), y.detach().view(torch.int32)), step
    assert [float(f) for f in c1.clipping_factors] == [float(f) for f in s1.clipping_factors]
  assert comp.iterations == 10 and len(comp.variables()) == 4
  assert all(0.0 < float(f) < 1.0 for f in c1.clipping_factors)


# ------------------------------------------------------------------------------------------------
# end to end
# ------------------------------------------------------------------------------------------------
def test_two_tower_model_trains_with_clippy_adagrad(tfrs):
  """test_gpu_api.py::test_two_tower_model_trains with ClippyAdagrad: the CUDA step tracks the oracle step by step."""
  torch.manual_seed(0)
  rng = np.random.RandomState(42)
  U, I, d, B = 2000, 2000, 64, 4096

  class TwoTower(tfrs.Model):

    def __init__(self):
      super().__init__()
      self.user_model = tfrs.layers.embedding.Embedding(U, d)
      self.item_model = tfrs.layers.embedding.Embedding(I, d)
      self.task = tfrs.tasks.Retrieval()

    def compute_loss(self, features, training=False):
      return self.task(self.user_model(features["user_id"]), self.item_model(features["movie_id"]),
                       compute_metrics=not training)

  kw = dict(var_rel=0.5, acc_rel=1e-2, abs_thr=1e-3)
  model = TwoTower()
  opt = tfrs.experimental.optimizers.ClippyAdagrad(0.5, variable_relative_threshold=kw["var_rel"],
                                                   accumulator_relative_threshold=kw["acc_rel"],
                                                   absolute_threshold=kw["abs_thr"], export_clipping_factors=True)
  model.compile(optimizer=opt)
  ut = model.user_model.weight.cpu().numpy().copy(); it = model.item_model.weight.cpu().numpy().copy()
  ua = np.full_like(ut, 0.1); ia = np.full_like(it, 0.1)
  losses = []
  uid = rng.randint(0, U, size=B).astype(np.int64); iid = rng.randint(0, I, size=B).astype(np.int64)
  for step in range(3):
    out = model.train_step({"user_id": cu(uid), "movie_id": cu(iid)})
    losses.append(float(out["loss"]))
    qe, ce = orc.gather(ut, uid), orc.gather(it, iid)
    np.testing.assert_allclose(losses[-1], orc.retrieval_loss(qe, ce), rtol=1e-5)
    dq, dc = orc.retrieval_loss_grads(qe, ce)
    ut, ua, uf = co.clippy_adagrad_sparse(ut, ua, uid, dq.astype(np.float32), 0.5, **kw)
    it, ia, itf = co.clippy_adagrad_sparse(it, ia, iid, dc.astype(np.float32), 0.5, **kw)
    np.testing.assert_allclose([float(f) for f in opt.clipping_factors], [uf, itf], rtol=1e-4)
    np.testing.assert_allclose(model.user_model.weight.cpu().numpy(), ut, rtol=1e-4, atol=2e-5)
    np.testing.assert_allclose(model.item_model.weight.cpu().numpy(), it, rtol=1e-4, atol=2e-5)
  assert losses[-1] < losses[0]
  assert opt.iterations == 3


def _synthetic_data(num_dense, vocab_sizes, dataset_size, batch_size, seed=0):
  """experimental/models/ranking_test.py:_generate_synthetic_data: labels = int((mean(dense) + sum(ids)/sum(vocab)) / 2 + 0.5)."""
  g = torch.Generator(device="cuda"); g.manual_seed(seed)
  dense = torch.rand((dataset_size, num_dense), generator=g, device="cuda")
  sparse = [torch.randint(0, v, (dataset_size,), generator=g, device="cuda", dtype=torch.int32) for v in vocab_sizes]
  labels = ((dense.mean(1) + torch.stack(sparse, -1).sum(1).float() / sum(vocab_sizes)) / 2.0 + 0.5).to(torch.int32)
  return [({"dense_features": dense[lo:lo + batch_size],
            "sparse_features": {str(i): s[lo:lo + batch_size] for i, s in enumerate(sparse)}}, labels[lo:lo + batch_size])
          for lo in range(0, dataset_size - batch_size + 1, batch_size)]


def test_ranking_model_trains_with_composite_optimizer(tfrs):
  vocab = [30, 3, 26]
  torch.manual_seed(1)
  model = tfrs.experimental.models.Ranking(
      embedding_layer=torch.nn.ModuleDict({str(i): tfrs.layers.embedding.Embedding(v, 16) for i, v in enumerate(vocab)}))
  clippy = tfrs.experimental.optimizers.ClippyAdagrad(0.1, export_clipping_factors=True)
  model.compile(optimizer=tfrs.experimental.optimizers.CompositeOptimizer([
      (clippy, lambda: model.embedding_trainable_variables),
      (tfrs.optimizers.Adagrad(0.05), lambda: model.dense_trainable_variables)]))
  data = _synthetic_data(8, vocab, 64, 16, seed=5)
  losses = [float(model.evaluate(data)["loss"])]
  for _ in range(15):
    model.fit(data, epochs=1)
    losses.append(float(model.evaluate(data)["loss"]))
  assert np.isfinite(losses).all() and losses[-1] < losses[0], losses
  assert model.optimizer.iterations == 15 * len(data)
  assert len(clippy.clipping_factors) == 3 and all(0.0 < float(f) <= 1.0 for f in clippy.clipping_factors)
  for p in model.parameters():
    assert torch.isfinite(p).all()
