"""GPU tests of TPUEmbedding (K11), PartialTPUEmbedding and SGD: bit for bit against the NumPy oracle
(embedding_bag_oracle.py), and the reference's own tests restated (layers/embedding/tpu_embedding_layer_test.py,
experimental/layers/embedding/partial_tpu_embedding_test.py, experimental/models/ranking_test.py:115-174 with the
size_threshold axis)."""
import itertools
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import embedding_bag_oracle as ebo  # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def tfrs():
  import recommenders_b200 as t
  return t


def _bags(rng, B, max_len, vocab, bad=True, empty=True):
  lens = rng.randint(0 if empty else 1, max_len + 1, size=B)
  sp = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
  vals = rng.randint(0, vocab, size=int(sp[-1])).astype(np.int64)
  if bad and vals.size:
    k = rng.rand(vals.size)
    vals[k < 0.05] = vocab + rng.randint(0, 5, size=int((k < 0.05).sum()))
    vals[k > 0.95] = -1 - rng.randint(0, 5, size=int((k > 0.95).sum()))
  return vals, sp


def _to_sparse(vals, sp, B, dtype):
  rows = np.repeat(np.arange(B), np.diff(sp))
  cols = np.arange(vals.size) - sp[rows]
  idx = torch.from_numpy(np.stack([rows, cols])).cuda()
  width = max(int(np.diff(sp).max(initial=0)), 1)
  return torch.sparse_coo_tensor(idx, torch.from_numpy(vals).to(dtype).cuda(), (B, width)).coalesce()


def _run(tfrs, fcs, feats, weights=None):
  """Forward under autograd, backward with a fixed gradient; (outputs, grads fed, {table index: (ids, rows)})."""
  layer = tfrs.layers.embedding.TPUEmbedding(fcs)
  outs = layer(feats, weights)
  flat = tfrs.layers.embedding.tpu_embedding_layer.flatten(outs)
  g = torch.Generator(device="cuda"); g.manual_seed(3)
  grads = [torch.randn(o.shape, generator=g, device="cuda") for o in flat]
  torch.autograd.backward(flat, grads)
  pairs = {}
  for i, t in enumerate(layer._tables):
    sg = t.pop_sparse_grads()
    assert len(sg) <= 1, "one (ids, rows) pair per table and call"
    if sg:
      pairs[i] = (sg[0][0].cpu().numpy(), sg[0][1].cpu().numpy())
  return layer, [o.detach() for o in flat], grads, pairs


@pytest.mark.parametrize("combiner,weighted,kind,dim", [c for c in itertools.product(
    ("sum", "mean", "sqrtn"), (False, True), ("ragged", "sparse", "dense"), (1, 3, 4, 16, 100, 128))
    if not (c[1] and c[2] == "dense")])   # dense inputs take no weights (test_dense_weights_raise)
def test_lookup_bit_exact(tfrs, combiner, weighted, kind, dim):
  rng = np.random.RandomState(dim * 7 + len(combiner))
  vocab, B = 50, 37
  tab = tfrs.layers.embedding.TableConfig(vocab, dim, combiner=combiner)
  fcs = {"a": tfrs.layers.embedding.FeatureConfig(tab), "b": tfrs.layers.embedding.FeatureConfig(tab)}
  feats, weights, spec = {}, {} if weighted else None, {}
  for name in ("a", "b"):
    if kind == "dense":
      vals = rng.randint(-3, vocab + 3, size=(B, 3)).astype(np.int64)
      feats[name], spec[name] = torch.from_numpy(vals).cuda(), (vals, None, None)
      continue
    vals, sp = _bags(rng, B, 9, vocab)
    w = rng.uniform(-1, 2, size=vals.size).astype(np.float32) if weighted else None
    dt = torch.int32 if name == "a" else torch.int64
    if kind == "ragged":
      feats[name] = (torch.from_numpy(vals).to(dt).cuda(), sp if name == "a" else torch.from_numpy(sp).cuda())
      if weighted:
        weights[name] = torch.from_numpy(w).cuda()
    else:
      feats[name] = _to_sparse(vals, sp, B, dt)
      if weighted:
        weights[name] = torch.sparse_coo_tensor(feats[name].indices(), torch.from_numpy(w).cuda(), feats[name].shape)
    spec[name] = (vals, sp, w)
  layer, outs, grads, pairs = _run(tfrs, fcs, feats, weights)
  table = layer._tables[0].weight.cpu().numpy()
  exp_rows, exp_ids = [], []
  for name, o, g in zip(("a", "b"), outs, grads):
    vals, sp, w = spec[name]
    exp, _ = ebo.lookup(table, vals, sp, w, combiner)
    assert o.cpu().numpy().tobytes() == exp.tobytes(), name
    exp_rows.append(ebo.lookup_bwd(table.shape, vals, g.cpu().numpy(), sp, w, combiner))
    exp_ids.append(vals.reshape(-1))
  ids, rows = pairs[0]
  np.testing.assert_array_equal(ids, np.concatenate(exp_ids))
  assert rows.tobytes() == np.concatenate(exp_rows).tobytes()


@pytest.mark.parametrize("L", [1, 3, 8])
@pytest.mark.parametrize("dim", [3, 16])
def test_sequence_features(tfrs, L, dim):
  rng = np.random.RandomState(L + dim)
  tab = tfrs.layers.embedding.TableConfig(40, dim)
  fcs = {"s": tfrs.layers.embedding.FeatureConfig(tab, max_sequence_length=L), "p": tfrs.layers.embedding.FeatureConfig(tab)}
  vals, sp = _bags(rng, 29, 6, 40)
  w = rng.uniform(0, 2, size=vals.size).astype(np.float32)
  feats = {"s": (torch.from_numpy(vals).cuda(), sp), "p": (torch.from_numpy(vals).cuda(), sp)}
  layer, outs, grads, pairs = _run(tfrs, fcs, feats, {"s": torch.from_numpy(w).cuda(), "p": None})
  table = layer._tables[0].weight.cpu().numpy()
  p_out, s_out = outs      # sorted keys: "p", "s"
  exp, _ = ebo.lookup(table, vals, sp, w, max_sequence_length=L)
  assert tuple(s_out.shape) == (29, L, dim) and s_out.cpu().numpy().tobytes() == exp.tobytes()
  exp_p, _ = ebo.lookup(table, vals, sp)
  assert p_out.cpu().numpy().tobytes() == exp_p.tobytes()
  rows = np.concatenate([ebo.lookup_bwd(table.shape, vals, grads[0].cpu().numpy(), sp),
                         ebo.lookup_bwd(table.shape, vals, grads[1].cpu().numpy(), sp, w, max_sequence_length=L)])
  assert pairs[0][1].tobytes() == rows.tobytes()


def test_long_bags_and_empty_batch(tfrs):
  rng = np.random.RandomState(5)
  for combiner in ("sum", "mean", "sqrtn"):
    tab = tfrs.layers.embedding.TableConfig(3000, 64, combiner=combiner)
    lens = np.array([1500, 0, 1, 2500, 1024])
    sp = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    vals = rng.randint(0, 3000, size=int(sp[-1]))
    w = rng.uniform(0, 1, size=vals.size).astype(np.float32)
    fcs = {"x": tfrs.layers.embedding.FeatureConfig(tab)}
    layer, outs, grads, pairs = _run(tfrs, fcs, {"x": (torch.from_numpy(vals).cuda(), sp)},
                                     {"x": torch.from_numpy(w).cuda()})
    table = layer._tables[0].weight.cpu().numpy()
    exp, _ = ebo.lookup(table, vals, sp, w, combiner)
    assert outs[0].cpu().numpy().tobytes() == exp.tobytes()
    assert pairs[0][1].tobytes() == ebo.lookup_bwd(table.shape, vals, grads[0].cpu().numpy(), sp, w, combiner).tobytes()
  layer = tfrs.layers.embedding.TPUEmbedding({"x": tfrs.layers.embedding.FeatureConfig(tab)})
  out = layer({"x": (torch.zeros(0, dtype=torch.int64, device="cuda"), np.zeros(1, np.int64))})
  assert tuple(out["x"].shape) == (0, 64)


def test_many_features_split_the_parameter_block(tfrs):
  rng = np.random.RandomState(9)
  tabs = [tfrs.layers.embedding.TableConfig(20 + k, 4 + (k % 3), combiner=("sum", "mean", "sqrtn")[k % 3]) for k in range(7)]
  fcs = [tfrs.layers.embedding.FeatureConfig(tabs[k % 7]) for k in range(300)]
  feats, spec = [], []
  for k in range(300):
    vals, sp = _bags(rng, 5, 4, 20 + k % 7)
    feats.append((torch.from_numpy(vals).cuda(), sp)); spec.append((vals, sp))
  before = tfrs.ops.launch_count()
  layer, outs, grads, pairs = _run(tfrs, fcs, feats)
  for k, (o, g) in enumerate(zip(outs, grads)):
    t = layer._tables[k % 7].weight.cpu().numpy()
    exp, _ = ebo.lookup(t, *spec[k], None, tabs[k % 7].combiner)
    assert o.cpu().numpy().tobytes() == exp.tobytes(), k
  for i in range(7):
    t = layer._tables[i].weight.cpu().numpy()
    rows = [ebo.lookup_bwd(t.shape, spec[k][0], grads[k].cpu().numpy(), spec[k][1], None, tabs[i].combiner)
            for k in range(i, 300, 7)]
    assert pairs[i][1].tobytes() == np.concatenate(rows).tobytes()
  assert tfrs.ops.launch_count() - before >= 2 * 3   # 300 features: three groups forward and backward


def test_one_launch_each_way(tfrs):
  rng = np.random.RandomState(2)
  tabs = [tfrs.layers.embedding.TableConfig(100, d) for d in (4, 8, 3)]
  fcs = {f"f{k}": tfrs.layers.embedding.FeatureConfig(tabs[k % 3]) for k in range(26)}
  feats = {}
  for k in range(26):
    vals, sp = _bags(rng, 64, 5, 100)
    feats[f"f{k}"] = (torch.from_numpy(vals).cuda(), torch.from_numpy(sp).cuda())
  layer = tfrs.layers.embedding.TPUEmbedding(fcs)
  torch.cuda.synchronize()
  c0 = tfrs.ops.launch_count()
  outs = layer(feats)
  c1 = tfrs.ops.launch_count()
  sum(o.sum() for o in outs.values()).backward()
  c2 = tfrs.ops.launch_count()
  assert c1 - c0 == 1 and c2 - c1 == 1, (c1 - c0, c2 - c1)


def test_sgd_bit_exact(tfrs):
  rng = np.random.RandomState(4)
  rows, d, n = 500, 12, 4000
  zipf = np.minimum(rng.zipf(1.3, size=n) - 1, rows + 3)       # hot ids repeat, some out of range
  ids = torch.from_numpy(zipf.astype(np.int64)).cuda()
  g = rng.normal(size=(n, d)).astype(np.float32)
  t0 = rng.normal(size=(rows, d)).astype(np.float32)
  table = torch.from_numpy(t0).cuda()
  tfrs.ops.sparse_sgd_(table, ids, torch.from_numpy(g).cuda(), 0.3)
  assert table.cpu().numpy().tobytes() == ebo.sgd_sparse(t0, zipf, g, 0.3).tobytes()
  ps = [torch.from_numpy(rng.normal(size=s).astype(np.float32)).cuda() for s in [(7,), (300, 5), (1,), (1025, 3)]]
  gs = [torch.randn_like(p) for p in ps]
  exp = [ebo.sgd_dense(p.cpu().numpy(), q.cpu().numpy(), 0.05) for p, q in zip(ps, gs)]
  tfrs.ops.sgd_dense_(ps, gs, 0.05)
  assert all(p.cpu().numpy().tobytes() == e.tobytes() for p, e in zip(ps, exp))


# ------------------------------------------------------------------------------------------------
# layers/embedding/tpu_embedding_layer_test.py restated
# ------------------------------------------------------------------------------------------------
VIDEO = np.arange(8, dtype=np.float32).reshape(2, 4)
USER = np.arange(8, dtype=np.float32).reshape(4, 2)
FIXTURE = {"watched": ([0, 0, 1, 0, 1, 1], [0, 1, 3, 5, 6]), "favorited": ([0, 1, 1, 0, 0, 1], [0, 2, 3, 4, 6]),
           "friends": ([3, 0, 1, 2, 3, 0, 1, 2], [0, 1, 4, 5, 8])}
ACTIVATIONS = {"watched": [[0, 1, 2, 3], [4, 6, 8, 10], [4, 6, 8, 10], [4, 5, 6, 7]],
               "favorited": [[4, 6, 8, 10], [4, 5, 6, 7], [0, 1, 2, 3], [4, 6, 8, 10]],
               "friends": [[6, 7], [2, 3], [6, 7], [2, 3]]}


def _fixture_layer(tfrs):
  init = lambda values: (lambda shape, device: torch.from_numpy(values).to(device))
  video = tfrs.layers.embedding.TableConfig(2, 4, initializer=init(VIDEO), combiner="sum", name="video_table")
  user = tfrs.layers.embedding.TableConfig(4, 2, initializer=init(USER), combiner="mean", name="user_table")
  fc = {"watched": tfrs.layers.embedding.FeatureConfig(video, name="watched"),
        "favorited": tfrs.layers.embedding.FeatureConfig(video, name="favorited"),
        "friends": tfrs.layers.embedding.FeatureConfig(user, name="friends")}
  return tfrs.layers.embedding.TPUEmbedding(fc, optimizer=None), video, user


def _fixture_inputs(sparse):
  out = {}
  for k, (vals, sp) in FIXTURE.items():
    vals, sp = np.array(vals), np.array(sp)
    out[k] = _to_sparse(vals, sp, 4, torch.int32) if sparse else (torch.tensor(vals, dtype=torch.int32).cuda(), sp)
  return out


@pytest.mark.parametrize("optimizer,training,sparse", list(itertools.product(("sgd", "adagrad", "adam"), (True, False),
                                                                              (True, False))))
def test_reference_fixture(tfrs, optimizer, training, sparse):
  layer, video, user = _fixture_layer(tfrs)
  opt = {"sgd": lambda: tfrs.optimizers.SGD(0.1), "adagrad": lambda: tfrs.optimizers.Adagrad(0.1),
         "adam": lambda: tfrs.optimizers.Adam(0.1)}[optimizer]().bind(layer)
  with torch.set_grad_enabled(training):
    acts = layer(_fixture_inputs(sparse))
  for k, v in ACTIVATIONS.items():
    assert acts[k].detach().cpu().numpy().tobytes() == np.array(v, np.float32).tobytes(), k
  if not training:
    return
  # loss = sum of all activations: every table row moves by the count of its pooled occurrences
  opt.zero_grad()
  layer._tables[0]._sparse_grads.clear(); layer._tables[1]._sparse_grads.clear()
  acts = layer(_fixture_inputs(sparse))
  sum(a.sum() for a in acts.values()).backward()
  opt.apply_gradients()
  tv, tu = layer.embedding_tables[video].weight.cpu().numpy(), layer.embedding_tables[user].weight.cpu().numpy()
  if optimizer == "sgd":
    ids_v = np.concatenate([FIXTURE["favorited"][0], FIXTURE["watched"][0]])   # sorted feature order
    ev = ebo.sgd_sparse(VIDEO, ids_v, np.ones((ids_v.size, 4), np.float32), 0.1)
    vals, sp = np.array(FIXTURE["friends"][0]), np.array(FIXTURE["friends"][1])
    gu = ebo.lookup_bwd((4, 2), vals, np.ones((4, 2), np.float32), sp, None, "mean")
    eu = ebo.sgd_sparse(USER, vals, gu, 0.1)
    assert tv.tobytes() == ev.tobytes() and tu.tobytes() == eu.tobytes()
  else:
    assert not np.array_equal(tv, VIDEO) and not np.array_equal(tu, USER)


# ------------------------------------------------------------------------------------------------
# experimental/layers/embedding/partial_tpu_embedding_test.py restated
# ------------------------------------------------------------------------------------------------
def _partial_config(tfrs):
  T, F = tfrs.layers.embedding.TableConfig, tfrs.layers.embedding.FeatureConfig
  return {"small_1": F(T(vocabulary_size=10, dim=4)), "small_2": F(T(vocabulary_size=15, dim=4)),
          "large_1": F(T(vocabulary_size=20, dim=4)), "large_2": F(T(vocabulary_size=25, dim=4))}


@pytest.mark.parametrize("threshold,n_keras,has_tpu", [(None, 4, False), (0, 0, True), (-1, 0, True), (17, 2, True)])
def test_partial_tpu_embedding(tfrs, threshold, n_keras, has_tpu):
  layer = tfrs.experimental.layers.embedding.PartialTPUEmbedding(_partial_config(tfrs), tfrs.optimizers.Adagrad(0.1),
                                                                 size_threshold=threshold)
  assert len(layer.keras_embedding_layers) == n_keras and (layer.tpu_embedding is not None) == has_tpu
  inputs = {k: torch.randint(0, 10, (8,), device="cuda") for k in _partial_config(tfrs)}
  out = layer(inputs)
  assert set(out) == set(inputs) and all(tuple(v.shape) == (8, 4) for v in out.values())
  for k, emb in layer.keras_embedding_layers.items():
    assert torch.equal(out[k], emb.weight[inputs[k]])


# ------------------------------------------------------------------------------------------------
# experimental/models/ranking_test.py:115-174 with PartialTPUEmbedding and its size_threshold axis
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("interaction,bottom,top,concat_dense,use_weights,threshold", list(itertools.product(
    ("dot", "cross"), ("default", "mlp"), ("default", "mlp"), (True, False), (True, False), (None, -1, 20))))
def test_ranking_with_partial_tpu_embedding(tfrs, interaction, bottom, top, concat_dense, use_weights, threshold):
  vocab = [30, 3, 26]
  torch.manual_seed(0)
  T, F = tfrs.layers.embedding.TableConfig, tfrs.layers.embedding.FeatureConfig
  fc = {str(i): F(T(vocabulary_size=v, dim=16)) for i, v in enumerate(vocab)}

  class ConcatCross(torch.nn.Module):
    def __init__(self):
      super().__init__()
      self.cross = tfrs.layers.feature_interaction.Cross()

    def forward(self, inputs):
      return self.cross(torch.cat(inputs, dim=1))

  model = tfrs.experimental.models.Ranking(
      embedding_layer=tfrs.experimental.layers.embedding.PartialTPUEmbedding(fc, None, size_threshold=threshold),
      bottom_stack=None if bottom == "default" else tfrs.layers.blocks.MLP(units=[40, 16]),
      feature_interaction=tfrs.layers.feature_interaction.DotInteraction() if interaction == "dot" else ConcatCross(),
      top_stack=None if top == "default" else tfrs.layers.blocks.MLP(units=[40, 20, 1], final_activation="sigmoid"),
      concat_dense=concat_dense)
  model.compile(optimizer=tfrs.optimizers.Adagrad(0.1))
  g = torch.Generator(device="cuda"); g.manual_seed(0)
  dense = torch.rand((64, 8), generator=g, device="cuda")
  sparse = [torch.randint(0, v, (64,), generator=g, device="cuda", dtype=torch.int32) for v in vocab]
  labels = ((dense.mean(1) + torch.stack(sparse, -1).sum(1).float() / sum(vocab)) / 2.0 + 0.5).to(torch.int32)
  weights = torch.rand((64, 1), generator=g, device="cuda") if use_weights else None
  data = []
  for lo in range(0, 64, 16):
    feats = {"dense_features": dense[lo:lo + 16], "sparse_features": {str(i): s[lo:lo + 16] for i, s in enumerate(sparse)}}
    data.append((feats, labels[lo:lo + 16]) if weights is None else (feats, labels[lo:lo + 16], weights[lo:lo + 16]))
  before = [t.weight.clone() for t in tfrs.optimizers.embedding_tables(model)]
  history = model.fit([data[i % len(data)] for i in range(5)], epochs=1)
  assert np.isfinite(float(history[-1]["loss"]))
  metrics = model.evaluate(data, return_dict=True)
  assert 0.0 <= metrics["accuracy"] <= 1.0 and np.isfinite(float(metrics["loss"]))
  tables = tfrs.optimizers.embedding_tables(model)
  assert len(tables) == 3 and len(model.embedding_trainable_variables) == 3
  assert all(not torch.equal(b, t.weight) for b, t in zip(before, tables))


def test_sgd_trains_under_compile_and_composite(tfrs):
  rng = np.random.RandomState(8)
  T, F = tfrs.layers.embedding.TableConfig, tfrs.layers.embedding.FeatureConfig
  torch.manual_seed(3)
  fc = {"a": F(T(50, 8, combiner="mean"))}
  vals, sp = _bags(rng, 16, 4, 50, bad=False)
  feats = {"a": (torch.from_numpy(vals).cuda(), sp)}

  def build():
    torch.manual_seed(3)
    emb = tfrs.layers.embedding.TPUEmbedding(fc)
    lin = torch.nn.Linear(8, 1).cuda()
    return emb, lin

  def step(emb, lin, opt):
    opt.zero_grad()
    loss = lin(emb(feats)["a"]).square().mean()
    loss.backward()
    opt.apply_gradients()

  e1, l1 = build()
  o1 = tfrs.optimizers.SGD(0.5).bind(torch.nn.ModuleList([e1, l1]))
  e2, l2 = build()
  m2 = torch.nn.ModuleList([e2, l2])
  o2 = tfrs.experimental.optimizers.CompositeOptimizer(
      [(tfrs.optimizers.SGD(0.5), lambda: list(e2._tables)), (tfrs.optimizers.SGD(0.5), lambda: list(l2.parameters()))]).bind(m2)
  for _ in range(3):
    step(e1, l1, o1); step(e2, l2, o2)
  assert torch.equal(e1._tables[0].weight, e2._tables[0].weight) and torch.equal(l1.weight, l2.weight)
