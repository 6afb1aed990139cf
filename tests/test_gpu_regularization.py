"""H100 tests of K23 (dropout) and K24 (batch normalization) against tests/regularization_oracle.py: dropout masks and
outputs bit for bit at every size, vector and grid edge, noise-shape pattern, rate and alignment; the layers' training
phase, launch counts, the keep fraction, seeding and attached masks; batch norm within 1e-5 of the oracle's max |value|
in both modes, with masks, shifted rows and odd widths, bitwise determinism; and two towers trained end to end with
torch's dropout and batch-norm ops banned."""
import itertools
import math

import numpy as np
import pytest
import torch

import regularization_oracle as ro
import recommenders_b200 as tfrs
from recommenders_b200 import backend, ops
from recommenders_b200.data import Dataset
from recommenders_b200.layers.blocks import Dense
from recommenders_b200.layers.embedding import Embedding
from test_gpu_gru import _SequentialModel, _histories

pytestmark = pytest.mark.gpu


def _cu(a, grad=False):
  if a is None:
    return None
  return torch.from_numpy(np.ascontiguousarray(a)).cuda().requires_grad_(grad)


def _check(name, got, exp, bar=1e-5, scale=None):
  got = got.detach().double().cpu().numpy() if isinstance(got, torch.Tensor) else np.asarray(got, np.float64)
  exp = np.asarray(exp, np.float64)
  assert got.shape == exp.shape, (name, got.shape, exp.shape)
  if scale is None:
    scale = max(float(np.abs(exp).max()) if exp.size else 0.0, 1e-30)
  err = float(np.abs(got - exp).max()) if exp.size else 0.0
  assert err <= bar * scale, f"{name}: max |err| {err:.3e} > {bar:g} * {scale:.3e}"


def _bits(t):
  return t.detach().cpu().numpy().view(np.uint32)


def _grid_threads():
  return torch.cuda.get_device_properties(0).multi_processor_count * 16 * 256


# ---- K23 dropout: bit-exact masks ---------------------------------------------------------------------------------
def test_dropout_sizes_match_the_oracle_bit_for_bit():
  edge = 4 * _grid_threads()   # elements one grid-stride pass covers in the vector kernel
  sizes = list(range(1, 10)) + [15, 16, 17, 1023, 1024, 1025, edge - 5, edge - 1, edge, edge + 1, edge + 4,
                                2 * edge + 3, (1 << 24) + 7]
  rng = np.random.RandomState(0)
  for n in sizes:
    x = rng.normal(size=n).astype(np.float32)
    y = ops.dropout(_cu(x), 0.3, 0x9E3779B97F4A7C15, n)
    assert np.array_equal(_bits(y), ro.dropout(x, 0.3, 0x9E3779B97F4A7C15, n).view(np.uint32)), n


@pytest.mark.parametrize("shape", [(37,), (6, 35), (3, 5, 33), (2, 3, 4, 9), (4, 1, 7, 5)])
def test_every_noise_shape_pattern_matches_the_oracle(shape):
  rng = np.random.RandomState(len(shape))
  x = rng.normal(size=shape).astype(np.float32)
  for flags in itertools.product((False, True), repeat=len(shape)):
    noise = tuple(1 if f else None for f in flags)
    call = int(rng.randint(0, 2**31)) << 20
    y = ops.dropout(_cu(x), 0.5, 77, call, noise)
    exp = ro.dropout(x, 0.5, 77, call, noise)
    assert np.array_equal(_bits(y), exp.view(np.uint32)), (shape, noise)


@pytest.mark.parametrize("rate", [0.0, 2.0**-24, 0.1, 0.5, 0.999])
def test_rates_match_the_oracle(rate):
  x = np.random.RandomState(1).normal(size=(300, 77)).astype(np.float32)
  for noise in (None, (300, 1)):
    y = ops.dropout(_cu(x), rate, 5, 2**40 + 3, noise)
    assert np.array_equal(_bits(y), ro.dropout(x, rate, 5, 2**40 + 3, noise).view(np.uint32))


def test_unaligned_and_strided_views_match_the_oracle():
  base = np.random.RandomState(2).normal(size=4099).astype(np.float32)
  xb = _cu(base)
  for off in (1, 2, 3):
    y = ops.dropout(xb[off:off + 4093], 0.25, 3, 1)
    assert np.array_equal(_bits(y), ro.dropout(base[off:off + 4093], 0.25, 3, 1).view(np.uint32))
  x2 = _cu(base[:4096].reshape(64, 64))
  y = ops.dropout(x2.t(), 0.25, 3, 1, (None, 1))
  exp = ro.dropout(np.ascontiguousarray(base[:4096].reshape(64, 64).T), 0.25, 3, 1, (None, 1))
  assert np.array_equal(_bits(y), exp.view(np.uint32))


def test_dropped_nan_and_inf_are_plus_zero():
  x = np.array([np.nan, np.inf, -np.inf, -0.0, -1.0] * 400, np.float32)
  y = ops.dropout(_cu(x), 0.5, 11, 0).cpu().numpy()
  exp = ro.dropout(x, 0.5, 11, 0)
  # a kept NaN stays NaN (its payload is the device's); every other element, +0 for the dropped ones, bit for bit
  nan = np.isnan(exp)
  assert np.array_equal(np.isnan(y), nan) and nan.any()
  assert np.array_equal(y[~nan].view(np.uint32), exp[~nan].view(np.uint32))


# ---- K23 dropout: the layers -------------------------------------------------------------------------------------
def test_the_backward_applies_the_same_mask():
  rng = np.random.RandomState(3)
  x, g = rng.normal(size=(8, 5, 6)).astype(np.float32), rng.normal(size=(8, 5, 6)).astype(np.float32)
  xt = _cu(x, True)
  layer = tfrs.layers.SpatialDropout1D(0.4, seed=21)
  y = layer(xt, training=True)
  y.backward(_cu(g))
  assert np.array_equal(_bits(y), ro.dropout(x, 0.4, 21, 0, (8, 1, 6)).view(np.uint32))
  assert np.array_equal(_bits(xt.grad), ro.dropout(g, 0.4, 21, 0, (8, 1, 6)).view(np.uint32))


def test_inference_rate_0_and_plain_calls_are_identities_without_launches():
  x = torch.randn((64, 32), device="cuda", requires_grad=True)
  d, z = tfrs.layers.Dropout(0.5), tfrs.layers.Dropout(0.0)
  n = ops.launch_count()
  assert d(x) is x and d(x, training=False) is x and z(x, training=True) is x
  with backend.learning_phase_scope(False):
    assert d(x) is x
  with backend.learning_phase_scope(True):
    assert z(x) is x
  assert ops.launch_count() == n
  with backend.learning_phase_scope(True):
    y = d(x)
  assert ops.launch_count() == n + 1 and y is not x
  y.sum().backward()
  assert ops.launch_count() == n + 2


def test_the_keep_fraction_is_within_6_sigma_of_the_binomial():
  n, rate = 1 << 24, 0.3
  y = tfrs.layers.Dropout(rate, seed=99)(torch.ones(n, device="cuda"), training=True)
  kept = int((y != 0).sum())
  p = 1 - ro.threshold(rate) / 2**24
  assert abs(kept - n * p) <= 6 * math.sqrt(n * p * (1 - p))


def test_successive_calls_differ_and_seeded_runs_repeat():
  x = torch.ones((128, 64), device="cuda")

  def run():
    torch.manual_seed(0)
    layer = tfrs.layers.Dropout(0.5)
    return [layer(x, training=True) for _ in range(3)]

  a, b = run(), run()
  assert not torch.equal(a[0], a[1]) and not torch.equal(a[1], a[2])
  for u, v in zip(a, b):
    assert torch.equal(u, v)


def test_the_attached_mask_survives_spatial_dropout_into_gru():
  torch.manual_seed(0)
  rng = np.random.RandomState(4)
  ids = rng.randint(1, 30, size=(16, 9))
  ids[rng.rand(16, 9) < 0.3] = 0
  idt = torch.from_numpy(ids).cuda()
  e = Embedding(30, 12, mask_zero=True)(idt)
  s = tfrs.layers.SpatialDropout1D(0.2, seed=4)(e, training=True)
  assert torch.equal(ops.attached_mask(s), ops.attached_mask(e))
  gru = tfrs.layers.GRU(8)
  h = gru(s)
  h_explicit = gru(s.clone(), mask=idt != 0)
  assert torch.equal(h, h_explicit)
  assert not torch.equal(h, gru(s.clone()))


def test_dropout_input_checks():
  with pytest.raises(NotImplementedError, match="rank 5"):
    ops.dropout(torch.zeros((1, 2, 1, 2, 2), device="cuda"), 0.5, 1, 0)
  with pytest.raises(TypeError, match="float32"):
    ops.dropout(torch.zeros(4, device="cuda", dtype=torch.float16), 0.5, 1, 0)
  with pytest.raises(ValueError, match="3-D"):
    tfrs.layers.SpatialDropout1D(0.5)(torch.zeros((2, 3), device="cuda"), training=True)
  with pytest.raises(ValueError, match="noise_shape"):
    tfrs.layers.Dropout(0.5, noise_shape=(2, 2))(torch.zeros((4, 3), device="cuda"), training=True)
  assert ops.dropout(torch.zeros((0, 3), device="cuda"), 0.5, 1, 0).shape == (0, 3)


# ---- K24 batch normalization -------------------------------------------------------------------------------------
def _bn_case(N, d, training, lead=None, offset=0.0, mask=None, center=True, scale=True, momentum=0.9,
             seed=0, masked_value=None):
  rng = np.random.RandomState(seed)
  shape = tuple(lead) + (d,) if lead else (N, d)
  x = (rng.normal(size=shape) + offset).astype(np.float32)
  if masked_value is not None:
    x[np.asarray(mask) == 0] = masked_value
  g = rng.normal(size=shape).astype(np.float32)
  gamma = rng.normal(size=d).astype(np.float32) if scale else None
  beta = rng.normal(size=d).astype(np.float32) if center else None
  mm = (rng.normal(size=d) + offset).astype(np.float32)
  mv = (rng.rand(d) + 0.5).astype(np.float32)
  xt, gt, bt = _cu(x, True), _cu(gamma, True), _cu(beta, True)
  mmt, mvt = _cu(mm), _cu(mv)
  mt = None if mask is None else _cu(mask)
  y = ops.batch_norm(xt, gt, bt, mmt, mvt, training, momentum, 1e-3, mt)
  (y * _cu(g)).sum().backward()
  ey, emm, emv = ro.batch_norm_forward(x, gamma, beta, mm, mv, training, momentum, 1e-3, mask)
  dx, dg, db = ro.batch_norm_backward(x, gamma, g, mm, mv, training, 1e-3, mask)
  _check("y", y, ey)
  # with two kept rows, xhat = +-sqrt(var / (var + eps)) whatever x is, and the training dx = gamma rstd (dy_0 - dy_1)
  # (1 - xhat^2) / 2 is what is left after terms of size gamma rstd dy cancel: fp32 is held to that size there
  two_rows = training and mask is None and x.reshape(-1, d).shape[0] == 2
  terms = np.abs(g).max() * (1.0 if gamma is None else np.abs(gamma).max()) / math.sqrt(float(np.float32(1e-3)))
  _check("dx", xt.grad, dx, scale=float(terms) if two_rows else None)
  if scale:
    _check("dgamma", gt.grad, dg)
  if center:
    _check("dbeta", bt.grad, db)
  _check("moving_mean", mmt, emm)
  _check("moving_variance", mvt, emv)


BN_SHAPES = [(1, 1), (1, 33), (2, 1), (7, 31), (33, 32), (100, 33), (257, 63), (1000, 64), (4097, 257), (3000, 1024),
             (65, 1023)]


@pytest.mark.parametrize("training", [True, False])
@pytest.mark.parametrize("N,d", BN_SHAPES)
def test_batch_norm_shapes_match_the_oracle(N, d, training):
  _bn_case(N, d, training, seed=N * 3 + d)


@pytest.mark.parametrize("training", [True, False])
@pytest.mark.parametrize("d", [1, 33])
def test_batch_norm_over_2_20_plus_1_rows(d, training):
  _bn_case((1 << 20) + 1, d, training, seed=d)


@pytest.mark.parametrize("training", [True, False])
@pytest.mark.parametrize("d", [1, 64, 1024])
def test_batch_norm_rows_with_mean_1e4_and_std_1(d, training):
  _bn_case(3000, d, training, offset=1e4, seed=d)


@pytest.mark.parametrize("training", [True, False])
def test_batch_norm_without_center_or_scale(training):
  _bn_case(200, 40, training, center=False, scale=False, seed=3)
  _bn_case(200, 40, training, center=False, seed=4)


@pytest.mark.parametrize("kind", [np.bool_, np.int32, np.int64])
@pytest.mark.parametrize("training", [True, False])
def test_batch_norm_with_a_passed_mask(kind, training):
  rng = np.random.RandomState(8)
  mask = (rng.rand(16, 50) < 0.7).astype(kind)
  _bn_case(0, 64, training, lead=(16, 50), mask=mask, seed=9)
  _bn_case(0, 33, training, lead=(16, 50), mask=mask, offset=1e4, seed=10)


@pytest.mark.parametrize("masked_value", [0.0, 1e6])
@pytest.mark.parametrize("d", [1, 33])
def test_masked_rows_far_from_the_kept_rows_do_not_move_the_moments(d, masked_value):
  # zero padding (or 1e6) next to kept rows with mean 1e4 and std 1: every 4th row dropped, and in the long case the
  # first rows of every chunk too, so no chunk can shift its sums by a dropped row
  mask = np.arange(8192) % 4 != 0
  _bn_case(8192, d, True, offset=1e4, mask=mask, masked_value=masked_value, seed=d)
  long = np.ones(1 << 18, bool)
  long[np.arange(1 << 18) % 1000 < 300] = False
  _bn_case(1 << 18, d, True, offset=1e4, mask=long, masked_value=masked_value, seed=d + 1)


@pytest.mark.parametrize("masked_value", [0.0, 1e6])
def test_a_chunk_whose_first_kept_row_is_past_its_first_256_rows(masked_value):
  # (65536, 512) runs 512-row chunks; rows 0-299 of every 1000 are dropped, so chunk 0 keeps its first row at 300
  mask = np.arange(1 << 16) % 1000 >= 300
  _bn_case(1 << 16, 512, True, offset=1e4, mask=mask, masked_value=masked_value, seed=5)


def test_the_moving_statistics_version_moves_with_them():
  bn = tfrs.layers.BatchNormalization()
  x = torch.randn((64, 8), device="cuda")
  bn(x)
  v = bn.moving_mean._version, bn.moving_variance._version
  bn(x)
  assert (bn.moving_mean._version, bn.moving_variance._version) == v
  bn(x, training=True)
  assert bn.moving_mean._version > v[0] and bn.moving_variance._version > v[1]


@pytest.mark.parametrize("training", [True, False])
def test_batch_norm_with_an_all_masked_batch(training):
  _bn_case(0, 20, training, lead=(4, 6), mask=np.zeros((4, 6), bool), seed=11)


def test_batch_norm_with_an_attached_mask():
  torch.manual_seed(0)
  rng = np.random.RandomState(12)
  ids = rng.randint(1, 40, size=(8, 11))
  ids[rng.rand(8, 11) < 0.4] = 0
  e = Embedding(40, 16, mask_zero=True)(torch.from_numpy(ids).cuda())
  bn = tfrs.layers.BatchNormalization(momentum=0.5)
  y = bn(e, training=True)
  assert torch.equal(ops.attached_mask(y), ops.attached_mask(e))
  ed = e.detach().cpu().numpy()
  ey, emm, emv = ro.batch_norm_forward(ed, np.ones(16), np.zeros(16), np.zeros(16), np.ones(16), True, 0.5, mask=ids)
  _check("y", y, ey)
  _check("moving_mean", bn.moving_mean, emm)
  _check("moving_variance", bn.moving_variance, emv)
  assert {n for n, _ in bn.named_buffers()} == {"moving_mean", "moving_variance"}
  assert {n for n, _ in bn.named_parameters()} == {"gamma", "beta"}
  assert "moving_mean" in bn.state_dict()


def test_batch_norm_determinism():
  rng = np.random.RandomState(13)
  x = rng.normal(size=(5000, 96)).astype(np.float32)

  def step():
    torch.manual_seed(0)
    bn = tfrs.layers.BatchNormalization()
    xt = _cu(x, True)
    y = bn(xt, training=True)
    (y * y).sum().backward()
    return [y.detach(), xt.grad, bn.gamma.grad, bn.beta.grad, bn.moving_mean, bn.moving_variance]

  for u, v in zip(step(), step()):
    assert torch.equal(u, v)
  for training in (True, False):
    mm, mv = torch.zeros(96, device="cuda"), torch.ones(96, device="cuda")
    mm2, mv2 = mm.clone(), mv.clone()
    g, b = torch.ones(96, device="cuda", requires_grad=True), torch.zeros(96, device="cuda", requires_grad=True)
    with torch.no_grad():
      y0 = ops.batch_norm(_cu(x), g, b, mm, mv, training)
    y1 = ops.batch_norm(_cu(x, True), g, b, mm2, mv2, training)
    assert torch.equal(y0, y1.detach()) and torch.equal(mm, mm2) and torch.equal(mv, mv2)


def test_batch_norm_launch_counts():
  x = torch.randn((300, 40), device="cuda", requires_grad=True)
  g, b = torch.ones(40, device="cuda", requires_grad=True), torch.zeros(40, device="cuda", requires_grad=True)
  mm, mv = torch.zeros(40, device="cuda"), torch.ones(40, device="cuda")
  for training, fwd, bwd in ((True, 3, 3), (False, 1, 2)):
    n = ops.launch_count()
    y = ops.batch_norm(x, g, b, mm, mv, training)
    assert ops.launch_count() - n == fwd
    n = ops.launch_count()
    y.sum().backward()
    assert ops.launch_count() - n == bwd


def test_batch_norm_input_checks():
  x = torch.zeros((4, 8), device="cuda")
  mm, mv = torch.zeros(8, device="cuda"), torch.ones(8, device="cuda")
  with pytest.raises(ValueError, match="two axes"):
    ops.batch_norm(torch.zeros(8, device="cuda"), None, None, mm, mv, True)
  with pytest.raises(ValueError, match="empty"):
    ops.batch_norm(torch.zeros((0, 8), device="cuda"), None, None, mm, mv, True)
  with pytest.raises(ValueError, match="gamma"):
    ops.batch_norm(x, torch.ones(7, device="cuda"), None, mm, mv, True)
  with pytest.raises(ValueError, match="mask"):
    ops.batch_norm(x, None, None, mm, mv, True, mask=torch.ones(3, dtype=torch.bool, device="cuda"))
  with pytest.raises(TypeError, match="mask"):
    ops.batch_norm(x, None, None, mm, mv, True, mask=torch.ones(4, device="cuda"))
  with pytest.raises(NotImplementedError, match="axis"):
    tfrs.layers.BatchNormalization(axis=0)(x)


# ---- end to end, torch's dropout and batch-norm ops banned --------------------------------------------------------
def _ban(monkeypatch, extra=()):
  def banned(*a, **k):
    raise AssertionError("a torch dropout / batch_norm / attention / softmax / layer_norm / matmul op ran")

  F = torch.nn.functional
  for mod, names in ((F, ("dropout", "dropout1d", "dropout2d", "alpha_dropout", "feature_alpha_dropout", "batch_norm",
                          "instance_norm", *extra)),
                     (torch, ("dropout", "dropout_", "feature_dropout", "alpha_dropout", "native_dropout",
                              "batch_norm", "native_batch_norm", "bernoulli")),
                     (torch.Tensor, ("bernoulli_", "bernoulli"))):
    for name in names:
      if hasattr(mod, name):
        monkeypatch.setattr(mod, name, banned)
  return banned


SASREC_DROPOUT_TOP10_FLOOR = 0.451  # half the held-out top-10 accuracy this seeded run reached on an H100 (0.9028)


class _SASRecDropout(torch.nn.Module):
  """test_gpu_attention's one-block SASRec tower with Dropout(0.2) on the embedding sum and on both residual
  branches."""

  def __init__(self, ids, T=10, d=32):
    super().__init__()
    self.lookup = tfrs.layers.StringLookup(vocabulary=ids, mask_token=None)
    self.item, self.position = Embedding(len(ids) + 1, d), Embedding(T, d)
    self.attention = tfrs.layers.MultiHeadAttention(2, 16)
    self.norm1, self.norm2 = tfrs.layers.LayerNormalization(), tfrs.layers.LayerNormalization()
    self.ff1, self.ff2 = Dense(64, activation="relu"), Dense(d)
    self.drop0, self.drop1, self.drop2 = (tfrs.layers.Dropout(0.2) for _ in range(3))

  def forward(self, history):
    ids = self.lookup(history)
    B, T = ids.shape
    x = self.drop0(self.item(ids) + self.position(torch.arange(T, device=ids.device).expand(B, T)))
    x = self.norm1(x + self.drop1(self.attention(x, x, use_causal_mask=True)))
    x = self.norm2(x + self.drop2(self.ff2(self.ff1(x))))
    return x[:, -1]


def test_sasrec_tower_with_dropout_trains_end_to_end(monkeypatch):
  banned = _ban(monkeypatch, ("scaled_dot_product_attention", "softmax", "layer_norm", "multi_head_attention_forward"))
  for name in ("softmax", "layer_norm", "bmm", "baddbmm", "matmul", "einsum"):
    monkeypatch.setattr(torch, name, banned)
  monkeypatch.setattr(torch.nn.MultiheadAttention, "forward", banned)

  ids, ctx, label = _histories()
  n_train = 49152
  torch.manual_seed(0)
  query_model = _SASRecDropout(ids)
  candidate_model = torch.nn.Sequential(tfrs.layers.StringLookup(vocabulary=ids, mask_token=None),
                                        Embedding(len(ids) + 1, 32))
  movies = Dataset.from_tensor_slices(ids)
  task = tfrs.tasks.Retrieval(metrics=tfrs.metrics.FactorizedTopK(candidates=movies.batch(128).map(candidate_model)))
  model = _SequentialModel(query_model, candidate_model, task)
  model.compile(optimizer=tfrs.optimizers.Adagrad(learning_rate=0.1))
  train = Dataset.from_tensor_slices({"context_movie_id": ctx[:n_train], "label_movie_id": label[:n_train]}).batch(1024)
  test = Dataset.from_tensor_slices({"context_movie_id": ctx[n_train:], "label_movie_id": label[n_train:]}).batch(2560)

  before = model.evaluate(test)
  hist = model.fit(train, epochs=3)
  assert query_model.drop0._calls == 3 * (n_train // 1024)   # one training call per batch, none in evaluate
  after = model.evaluate(test)
  again = model.evaluate(test)
  top10 = float(after["factorized_top_k/top_10_categorical_accuracy"])
  print(f"sequential tutorial (SASRec + dropout): loss {float(before['loss']):.4f} -> {float(after['loss']):.4f}, "
        f"held-out top-10 accuracy {float(before['factorized_top_k/top_10_categorical_accuracy']):.4f} -> {top10:.4f}")
  assert all(np.isfinite(float(h["loss"])) for h in hist)
  assert float(after["loss"]) < float(before["loss"])
  assert top10 >= SASREC_DROPOUT_TOP10_FLOOR
  assert query_model.drop0._calls == 3 * (n_train // 1024)
  for k in after:
    assert torch.equal(torch.as_tensor(after[k]), torch.as_tensor(again[k])), k


class _RankingModel(tfrs.Model):
  def __init__(self):
    super().__init__()
    self.tower = torch.nn.Sequential(Dense(256, activation="relu"), tfrs.layers.BatchNormalization(),
                                     tfrs.layers.Dropout(0.3), Dense(64, activation="relu"), Dense(1))
    self.task = tfrs.tasks.Ranking(loss=tfrs.losses.MeanSquaredError(),
                                   metrics=[tfrs.metrics.RootMeanSquaredError()])

  def compute_loss(self, features, training=False):
    return self.task(features["rating"], self.tower(features["x"]))


def test_ranking_tower_with_batch_norm_and_dropout_trains_end_to_end(monkeypatch):
  _ban(monkeypatch)
  rng = np.random.RandomState(0)
  n, f = 40960, 24
  x = rng.normal(size=(n, f)).astype(np.float32) * 3 + 2
  w = rng.normal(size=f) / math.sqrt(f)
  rating = np.clip(3 + np.tanh(x @ w - 2 * w.sum()) * 2 + rng.normal(size=n) * 0.3, 1, 5).astype(np.float32)[:, None]
  data = {"x": torch.from_numpy(x).cuda(), "rating": torch.from_numpy(rating).cuda()}
  n_train = 32768
  train = Dataset.from_tensor_slices({k: v[:n_train] for k, v in data.items()}).batch(1024)
  test = Dataset.from_tensor_slices({k: v[n_train:] for k, v in data.items()}).batch(2048)
  torch.manual_seed(0)
  model = _RankingModel()
  model.compile(optimizer=tfrs.optimizers.Adam(learning_rate=1e-3))
  before = float(model.evaluate(test)["root_mean_squared_error"])
  bn = model.tower[1]
  mm0, mv0 = bn.moving_mean.clone(), bn.moving_variance.clone()
  model.fit(train, epochs=3)
  assert not torch.equal(mm0, bn.moving_mean) and not torch.equal(mv0, bn.moving_variance)
  mm1, mv1 = bn.moving_mean.clone(), bn.moving_variance.clone()
  after = float(model.evaluate(test)["root_mean_squared_error"])
  assert torch.equal(mm1, bn.moving_mean) and torch.equal(mv1, bn.moving_variance)
  print(f"ranking tower (BatchNormalization + Dropout): held-out RMSE {before:.4f} -> {after:.4f}")
  assert np.isfinite(after) and after < before
  assert all(p is not bn.moving_mean for p in tfrs.optimizers.dense_variables(model))
