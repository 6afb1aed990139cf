"""UnifiedEmbedding on the GPU (K8): the reference's unified_embedding_test.py restated, the hashing and the lookups
bit-exact with the C oracle (tests/unified_oracle.c), the sparse gradients and one optimizer step on them, launch
counts, training, and errors."""
import numpy as np
import pytest
import torch

import clippy_oracle as co
import unified_oracle as uo

pytestmark = pytest.mark.gpu

INT64_MIN, INT64_MAX = -2**63, 2**63 - 1
INT32_MIN, INT32_MAX = -2**31, 2**31 - 1


@pytest.fixture(scope="module")
def tfrs():
  import recommenders_b200 as t
  from recommenders_b200.layers.feature_multiplexing import unified_embedding  # noqa: F401  (the tutorial's import)
  return t


def _ue():
  from recommenders_b200.layers.feature_multiplexing import unified_embedding
  return unified_embedding


def _dataset():
  """unified_embedding_test.py:setUp, draw for draw (including "city" drawn from the genre vocabulary); the ragged
  history is a (values, row_splits) pair."""
  rng = np.random.default_rng(seed=42)
  vocabs = {"genre": ["romance", "drama", "fantasy", "action", "comedy", "horror"],
            "year": [str(n) for n in range(1950, 2023)],
            "city": ["New York", "Los Angeles", "Chicago", "Houston", "Phoenix"],
            "history": [f"Movie {n}" for n in range(1000)],
            "label": [0, 1]}
  n = 10
  ds = {"genre": rng.choice(vocabs["genre"], size=n), "year": rng.choice(vocabs["year"], size=n),
        "city": rng.choice(vocabs["genre"], size=n), "num_watched": 100 * (1.0 - rng.power(4, size=n)).astype(int),
        "history": rng.choice(vocabs["history"], size=[n, 4]), "label": rng.choice(vocabs["label"], size=n)}
  lens = rng.integers(1, 10, size=n)
  ragged = [rng.choice(vocabs["history"], size=k) for k in lens]
  ds["history_varlen"] = (np.concatenate(ragged), np.concatenate([[0], np.cumsum(lens)]).astype(np.int64))
  return ds


def _layer(name, num_tables, features, buckets=10, dim=8, **kw):
  ue = _ue()
  cfg = ue.UnifiedEmbeddingConfig(buckets_per_table=buckets, dim_per_table=dim, num_tables=num_tables, name=name, **kw)
  for f, c in features:
    cfg.add_feature(f, c)
  return ue.UnifiedEmbedding(cfg, None)


def _tables(layer):
  return [t.weight.cpu().numpy() for t in layer._tables]


def _host(features):
  np_ = lambda v: v.cpu().numpy() if isinstance(v, torch.Tensor) else v
  return {k: (np_(v[0]), np_(v[1])) if isinstance(v, tuple) else np_(v) for k, v in features.items()}


def _check_forward(layer, features, spec, name, combiner="mean"):
  with torch.no_grad():
    outs = layer(features)
  exp, _ = uo.forward(_host(features), spec, _tables(layer), name, combiner)
  assert len(outs) == len(exp)
  for o, e in zip(outs, exp):
    assert tuple(o.shape) == e.shape
    np.testing.assert_array_equal(o.cpu().numpy(), e)
  return outs


# ---- the six tests of unified_embedding_test.py -----------------------------------------------------------------------
def test_single_feature(tfrs):
  spec = [("genre", 2)]
  out = _check_forward(_layer("single_ue_table", 1, spec), _dataset(), spec, "single_ue_table")[0]
  assert list(out.shape) == [10, 16]


@pytest.mark.parametrize("name,spec,widths", [
    ("multiple_ue_table", [("genre", 1), ("year", 2), ("city", 3)], [8, 16, 24]),
    ("reordered_ue_table", [("year", 2), ("genre", 1), ("city", 3)], [16, 8, 24]),   # test_feature_output_order
])
def test_multiple_features(tfrs, name, spec, widths):
  outs = _check_forward(_layer(name, 3, spec), _dataset(), spec, name)
  assert [list(o.shape) for o in outs] == [[10, w] for w in widths]


def test_dense_multivalent(tfrs):
  spec = [("history", 3)]
  out = _check_forward(_layer("dense_multivalent_ue_table", 3, spec), _dataset(), spec, "dense_multivalent_ue_table")[0]
  assert list(out.shape) == [10, 4, 24]


def test_sparse_multivalent(tfrs):
  spec = [("history_varlen", 3)]
  out = _check_forward(_layer("sparse_multivalent_ue_table", 3, spec), _dataset(), spec, "sparse_multivalent_ue_table")[0]
  assert list(out.shape) == [10, 24]


def test_save_model(tfrs):
  ds = _dataset()
  spec = [("year", 1), ("city", 3), ("genre", 2)]
  ue_layer = _layer("ue_table", 4, spec)
  mlp = tfrs.layers.blocks.MLP([16, 1], final_activation="sigmoid")
  with torch.no_grad():
    pred = mlp(torch.cat(ue_layer(ds), -1))
    ue2 = _ue().UnifiedEmbedding.from_config(ue_layer.get_config())
    ue2.load_state_dict(ue_layer.state_dict())
    mlp2 = tfrs.layers.blocks.MLP([16, 1], final_activation="sigmoid")
    mlp2(torch.zeros((1, 48), device="cuda"))
    mlp2.load_state_dict(mlp.state_dict())
    pred2 = mlp2(torch.cat(ue2(ds), -1))
  assert ue2.get_config() == ue_layer.get_config()
  assert list(pred.shape) == [10, 1]
  assert torch.equal(pred, pred2)


# ---- hashing ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("num_bins", [1, 3, 12_884_901_893])       # the last is a non-power-of-two above 2^33
def test_hash_bins_integers(tfrs, num_bins):
  rng = np.random.default_rng(1)
  edges = [0, 1, -1, 9, 10, -10, 999_999_999, 1_000_000_000, -1_000_000_000]
  v64 = np.concatenate([np.array(edges + [INT64_MIN, INT64_MAX, INT64_MIN + 1], np.int64),
                        rng.integers(INT64_MIN, INT64_MAX, size=200_000, dtype=np.int64),
                        rng.integers(-10**6, 10**6, size=50_000)])
  v32 = np.concatenate([np.array(edges + [INT32_MIN, INT32_MAX], np.int32),
                        rng.integers(INT32_MIN, INT32_MAX, size=100_000, dtype=np.int32)])
  for v, salt in ((v64, [7, 2**64 - 1]), (v32, 133)):
    got = tfrs.ops.hash_bins(torch.from_numpy(v).cuda(), num_bins, salt).cpu().numpy()
    np.testing.assert_array_equal(got, uo.hash_bins(v.astype(np.int64), num_bins, salt))


def test_hash_bins_strings(tfrs):
  rng = np.random.default_rng(2)
  strs = [rng.integers(0, 256, size=k, dtype=np.uint8).tobytes() for k in range(41) for _ in range(8)]
  strs += [bytes(rng.integers(0, 256, size=1024, dtype=np.uint8)), "日本語 héllo".encode()]
  data, off = uo.pack(strs)
  for num_bins, salt in ((1, 0), (3, [1, 2]), (12_884_901_893, [5, 9])):
    got = tfrs.ops.hash_bins((torch.from_numpy(data).cuda(), torch.from_numpy(off).cuda()), num_bins, salt).cpu().numpy()
    np.testing.assert_array_equal(got, uo.hash_bins(strs, num_bins, salt))
  # the API documentation examples
  d, o = uo.pack(["Hello", "TF"])
  assert tfrs.ops.hash_bins((torch.from_numpy(d).cuda(), torch.from_numpy(o).cuda()), 3, [1, 2]).tolist() == [2, 0]


# ---- forward ---------------------------------------------------------------------------------------------------------
def _mixed_features(rng, B=300, L=5):
  lens = rng.integers(0, 7, size=B)
  lens[:3] = 0                                                   # empty bags
  splits = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
  words = np.array(["", "a", "zürich", "x" * 30] + [f"w{k}" for k in range(50)])
  return {
      "uid": torch.from_numpy(rng.integers(-10**12, 10**12, size=B)).cuda(),                       # dense [B] int64
      "hist": torch.from_numpy(rng.integers(0, 1000, size=(B, L)).astype(np.int32)).cuda(),        # dense [B, L] int32
      "bag": (torch.from_numpy(rng.integers(0, 500, size=int(splits[-1]))).cuda(), torch.from_numpy(splits).cuda()),
      "tags": (rng.choice(words, size=int(splits[-1])), splits),                                    # ragged strings
      "city": rng.choice(words, size=B),                                                          # dense strings
      "unused": torch.zeros(3, device="cuda", dtype=torch.float32),
  }


@pytest.mark.parametrize("combiner", ["mean", "sum", "sqrtn"])
def test_forward_mixed_inputs_every_combiner(tfrs, combiner):
  rng = np.random.default_rng(3)
  feats = _mixed_features(rng)
  spec = [("uid", 2), ("hist", 3), ("bag", 2), ("tags", 1), ("city", 12)]
  layer = _layer("mix", 3, spec, buckets=997, dim=16, combiner=combiner)
  a = _check_forward(layer, feats, spec, "mix", combiner)
  with torch.no_grad():
    b = layer(feats)
  assert all(torch.equal(x, y) for x, y in zip(a, b))          # two runs, identical bits
  assert list(a[1].shape) == [300, 5, 48] and list(a[4].shape) == [300, 192]


@pytest.mark.parametrize("dist", ["uniform", "zipf"])
def test_forward_bench_shape(tfrs, dist):
  """The bench's cfg5 shape: 26 int64 features x 2 chunks over 4 tables of 13M x 16, B = 65536.  Bucket ids from the
  oracle, rows compared against the tables."""
  B, F = 65536, 26
  rng = np.random.default_rng(7)
  ids = [rng.integers(0, 1_000_000, size=B) if dist == "uniform" else np.minimum(rng.zipf(1.05, size=B) - 1, 999_999)
         for _ in range(F)]
  spec = [(f"f{k}", 2) for k in range(F)]
  layer = _layer("cfg5", 4, spec, buckets=13_000_000, dim=16)
  feats = {f"f{k}": torch.from_numpy(ids[k].astype(np.int64)).cuda() for k in range(F)}
  with torch.no_grad():
    outs = layer(feats)
    again = layer(feats)
  for (feat, chunks), o, o2, v in zip(uo.plan(spec, 4, "cfg5"), outs, again, ids):
    assert torch.equal(o, o2)
    for c, t, salt, pos in chunks:
      b = torch.from_numpy(uo.hash_bins(v, 13_000_000, salt)).cuda()
      assert torch.equal(o[:, pos * 16:(pos + 1) * 16], layer._tables[t].weight[b])
  del layer, outs, again
  torch.cuda.empty_cache()


# ---- backward and one optimizer step ---------------------------------------------------------------------------------
@pytest.mark.parametrize("combiner", ["mean", "sum", "sqrtn"])
def test_backward_pairs_and_optimizer_steps(tfrs, combiner):
  rng = np.random.default_rng(4)
  feats = _mixed_features(rng, B=200)
  spec = [("uid", 2), ("hist", 3), ("bag", 2), ("tags", 1), ("city", 3)]
  layer = _layer("bw", 4, spec, buckets=500, dim=8, combiner=combiner)
  tables0 = _tables(layer)
  outs = layer(feats)
  grads = [torch.from_numpy(rng.standard_normal(o.shape).astype(np.float32)).cuda() for o in outs]
  torch.autograd.backward(outs, grads)
  host = _host(feats)
  _, exp_ids = uo.forward(host, spec, tables0, "bw", combiner)
  exp_rows = uo.backward(host, spec, 4, 8, "bw", [g.cpu().numpy() for g in grads], combiner)
  pairs = {}
  for t, tab in enumerate(layer._tables):
    got = tab._sparse_grads
    assert len(got) == (1 if t in exp_ids else 0)
    if got:
      ids, rows = got[0]
      np.testing.assert_array_equal(ids.cpu().numpy(), exp_ids[t])
      np.testing.assert_array_equal(rows.cpu().numpy(), exp_rows[t])
      pairs[t] = (ids, rows)
  # one Adagrad step on those pairs
  opt = tfrs.optimizers.Adagrad(0.5).bind(layer)
  opt.apply_gradients()
  from oracle import oracle as orc
  for t, (ids, rows) in pairs.items():
    et, ea = orc.sparse_adagrad(tables0[t], np.full_like(tables0[t], 0.1), ids.cpu().numpy(), rows.cpu().numpy(), 0.5)
    np.testing.assert_array_equal(layer._tables[t].weight.cpu().numpy(), et)
  # and one ClippyAdagrad step after a fresh forward / backward
  tables1 = _tables(layer)
  outs = layer(feats)
  torch.autograd.backward(outs, grads)
  pairs = {t: tuple(x.cpu().numpy() for x in tab._sparse_grads[0]) for t, tab in enumerate(layer._tables) if tab._sparse_grads}
  clippy = tfrs.experimental.optimizers.ClippyAdagrad(0.1).bind(layer)
  clippy.apply_gradients()
  for t, (ids, rows) in pairs.items():
    et, _, _ = co.clippy_adagrad_sparse(tables1[t], np.full_like(tables1[t], 0.1), ids, rows, 0.1)
    np.testing.assert_array_equal(layer._tables[t].weight.cpu().numpy(), et)


# ---- launches --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n_features,ragged", [(1, False), (26, False), (26, True)])
def test_launch_counts(tfrs, n_features, ragged):
  B = 1024
  spec = [(f"f{k}", 2) for k in range(n_features)]
  layer = _layer("lc", 3, spec, buckets=1000, dim=16)
  feats = {f"f{k}": torch.randint(0, 10**6, (B,), device="cuda") for k in range(n_features)}
  if ragged:
    feats["f0"] = (torch.randint(0, 10**6, (3 * B,), device="cuda"), torch.arange(0, 3 * B + 1, 3, device="cuda"))
  torch.cuda.synchronize()
  n0 = tfrs.ops.launch_count()
  outs = layer(feats)
  n1 = tfrs.ops.launch_count()
  torch.autograd.backward(outs, [torch.ones_like(o) for o in outs])
  n2 = tfrs.ops.launch_count()
  assert n1 - n0 == (2 if ragged else 1)
  assert n2 - n1 == 1


def test_training_calls_free_their_outputs(tfrs):
  """A training call's outputs, bucket ids and uploads are freed once backward ran and the caller dropped them: the
  autograd node keeps no reference to the tensors it returns (with several outputs such a cycle is never collected)."""
  import gc
  import weakref
  rng = np.random.default_rng(6)
  feats = _mixed_features(rng, B=256)
  layer = _layer("leak", 3, [("uid", 2), ("hist", 1), ("bag", 2), ("tags", 1), ("city", 1)], buckets=1000, dim=8)
  for _ in range(2):                                   # the first call warms the caching allocator
    outs = layer(feats)
    refs = [weakref.ref(o._base if o._base is not None else o) for o in outs]
    torch.autograd.backward(outs, [torch.ones_like(o) for o in outs])
    pairs = [t.pop_sparse_grads() for t in layer._tables]
    id_refs = [weakref.ref(ids) for p in pairs for ids, _ in p]
    torch.cuda.synchronize()
    before = torch.cuda.memory_allocated()
    del outs, pairs
    gc.collect()
    assert all(r() is None for r in refs + id_refs)
  assert torch.cuda.memory_allocated() < before


# ---- training --------------------------------------------------------------------------------------------------------
def _movie_batches(rng, n_batches, B):
  """Six string features of the tutorial's shape; the label depends on the user and the movie."""
  out = []
  for _ in range(n_batches):
    uid, mid = rng.integers(0, 200, size=B), rng.integers(0, 300, size=B)
    feats = {"movie_id": np.char.mod("%d", mid), "user_id": np.char.mod("%d", uid),
             "user_gender": np.where(uid % 2 == 0, "True", "False"), "user_zip_code": np.char.mod("%05d", uid * 37 % 1000),
             "user_occupation_text": np.array(["doctor", "artist", "student", "other"])[uid % 4],
             "bucketized_user_age": np.char.mod("%d", 18 + uid % 5 * 7)}
    label = torch.from_numpy(((uid + mid) % 3 == 0).astype(np.float32)).cuda().reshape(-1, 1)
    out.append((feats, label))
  return out


def test_tutorial_model_trains(tfrs):
  torch.manual_seed(0)
  names = ["movie_id", "user_id", "user_gender", "user_zip_code", "user_occupation_text", "bucketized_user_age"]
  ue = _layer("unified_table", 2, [(n, 2) for n in names], buckets=500, dim=8)

  class UnifiedEmbeddingModel(tfrs.models.Model):
    def __init__(self):
      super().__init__()
      self.embedding = ue
      self.network = tfrs.layers.blocks.MLP([128, 64, 1], final_activation="sigmoid")
      self.task = tfrs.tasks.Ranking(metrics=[tfrs.metrics.AUC(name="AUC")])

    def compute_loss(self, inputs, training=False):
      feats, labels = inputs
      return self.task(labels, self.network(torch.cat(self.embedding(feats), -1)))

  model = UnifiedEmbeddingModel()
  model.compile(optimizer=tfrs.optimizers.Adagrad(0.1))
  data = _movie_batches(np.random.default_rng(5), 50, 256)
  losses = [float(model.train_step(b)["loss"]) for b in data]
  assert np.isfinite(losses).all()
  assert np.mean(losses[-5:]) < np.mean(losses[:5]), losses
  assert all(t._sparse_grads == [] for t in ue._tables)


def test_ranking_model_with_unified_embedding_trains(tfrs):
  torch.manual_seed(1)
  ue = _layer("rk", 2, [("a", 2), ("b", 2), ("c", 2)], buckets=100, dim=8)   # three [B, 16] embeddings
  model = tfrs.experimental.models.Ranking(embedding_layer=ue, bottom_stack=tfrs.layers.blocks.MLP([32, 16],
                                                                                                  final_activation="relu"))
  assert model.embedding_trainable_variables == [t.weight for t in ue._tables]
  model.compile(optimizer=tfrs.experimental.optimizers.CompositeOptimizer([
      (tfrs.experimental.optimizers.ClippyAdagrad(0.1), lambda: model.embedding_trainable_variables),
      (tfrs.optimizers.Adagrad(0.05), lambda: model.dense_trainable_variables)]))
  g = torch.Generator(device="cuda"); g.manual_seed(3)
  data = []
  for _ in range(4):
    dense = torch.rand((32, 8), generator=g, device="cuda")
    sp = {k: torch.randint(0, 30, (32,), generator=g, device="cuda") for k in "abc"}
    labels = ((dense.mean(1) + sum(sp.values()).float() / 90.0) / 2.0 + 0.5).to(torch.int32)
    data.append(({"dense_features": dense, "sparse_features": sp}, labels))
  losses = [float(model.evaluate(data)["loss"])]
  for _ in range(15):
    model.fit(data, epochs=1)
    losses.append(float(model.evaluate(data)["loss"]))
  assert np.isfinite(losses).all() and losses[-1] < losses[0], losses


# ---- errors ----------------------------------------------------------------------------------------------------------
def test_errors(tfrs):
  layer = _layer("err", 1, [("a", 1)])
  with pytest.raises(KeyError):
    layer({"b": torch.zeros(3, dtype=torch.int64, device="cuda")})
  with pytest.raises(TypeError):
    layer({"a": torch.zeros(3, device="cuda")})
  with pytest.raises(TypeError):
    layer({"a": torch.zeros(3, dtype=torch.bool, device="cuda")})
  with pytest.raises(RuntimeError, match="CUDA"):
    layer({"a": torch.zeros(3, dtype=torch.int64)})
  with pytest.raises(TypeError):
    layer({"a": []})
  with pytest.raises(ValueError, match="no bag"):                  # pooled values with row_splits = [0]
    layer({"a": (torch.arange(3, device="cuda"), np.array([0]))})


def test_empty_batch(tfrs):
  layer = _layer("empty", 2, [("a", 2), ("b", 1)])
  feats = {"a": torch.zeros(0, dtype=torch.int64, device="cuda"),
           "b": (torch.zeros(0, dtype=torch.int64, device="cuda"), np.array([0, 0, 0]))}
  outs = layer(feats)
  assert [list(o.shape) for o in outs] == [[0, 16], [2, 8]]
  assert not outs[1].any()
  torch.autograd.backward(outs, [torch.ones_like(o) for o in outs])
  assert all(ids.numel() == 0 for t in layer._tables for ids, _ in t.pop_sparse_grads())
