"""K13 (csrc/listwise.cu) on the GPU against tests/listwise_oracle.py: per-list losses, reduced losses, gradients and NDCG for
every loss x reduction x weighting, list lengths across the bitonic and packing edges, padding and other edge inputs,
determinism, NDCGMetric, and a restatement of the reference's listwise_ranking tutorial."""
import numpy as np
import pytest
import torch

import listwise_oracle as lo

pytestmark = pytest.mark.gpu

MODES = {"listmle": lo.LISTMLE, "hinge": lo.HINGE, "softmax": lo.SOFTMAX}
REDS = {"none": lo.RED_NONE, "sum": lo.RED_SUM, "auto": lo.RED_AUTO}
F32 = np.float32


@pytest.fixture(scope="module")
def tfrs():
  import recommenders_b200 as t
  return t


def _data(B, L, seed=0, pad=0.2, labels=5, scale=3.0, offset=None):
  rng = np.random.default_rng(seed)
  pred = (rng.normal(size=(B, L)) * scale).astype(F32)
  if offset is not None:
    pred = (pred + offset * rng.choice([-1.0, 1.0], size=(B, 1))).astype(F32)
  y = rng.integers(0, labels, size=(B, L)).astype(F32)
  y[rng.random((B, L)) < pad] = -1.0
  w = rng.uniform(0.25, 2.0, size=B).astype(F32)
  return pred, y, w


def _run(tfrs, mode, pred, y, w, red, T=1.0, seed=0, call=0, topn=None, g=None):
  ops = tfrs.ops
  p = torch.tensor(pred, device="cuda", requires_grad=True)
  stats = ops.ndcg_stats_buffer(p.device)
  out = ops.listwise_loss(p, torch.tensor(y, device="cuda"), None if w is None else torch.tensor(w, device="cuda"), mode, red, T,
                          seed, call, stats, topn)
  if g is None:
    g = np.ones(out.shape, F32) if red == lo.RED_NONE else F32(1.0)
  out.backward(torch.tensor(g, device="cuda"))
  return out.detach().cpu().numpy(), p.grad.cpu().numpy(), stats.cpu().numpy(), np.asarray(g, F32)


def _check(tfrs, mode, pred, y, w, red, T=1.0, seed=0, call=0, topn=None, g=None, ndcg=True):
  B, L = pred.shape
  out, dx, stats, g = _run(tfrs, mode, pred, y, w, red, T, seed, call, topn, g)
  wv = np.ones(B, F32) if w is None else np.asarray(w, F32).reshape(-1)
  l64, g64, Tb, n = lo.forward64(mode, pred, y, wv, T, seed, call)
  c = g.reshape(-1) if red == lo.RED_NONE else np.full(B, (F32(g) / F32(B)) if red == lo.RED_AUTO else F32(g), F32)
  inv_t = F32(1.0 / T)
  if mode == lo.HINGE:
    l32, dl32, _ = lo.hinge32(lo.scaled(pred, T), y, wv)
    per = (wv * l32).astype(F32)
    if red == lo.RED_NONE:
      assert np.array_equal(out.view(np.uint32), per.view(np.uint32))
    else:
      assert out.view(np.uint32) == np.asarray(lo.reduce_loss(per, B, L, red)).view(np.uint32)
    assert np.array_equal(dx.view(np.uint32), lo.backward32(dl32, g, red, T).view(np.uint32))
  else:
    lb, gb = lo.listmle_bars(l64, g64, Tb, n, wv) if mode == lo.LISTMLE else lo.softmax_bars(l64, g64, Tb, n, y, wv)
    ref = wv.astype(np.float64) * l64
    if red == lo.RED_NONE:
      assert lo.within(out, ref, lb)
    else:
      div = B if red == lo.RED_AUTO else 1
      assert lo.within(out, ref.sum() / div, lb.sum() / div + 2.0 ** -23 * abs(ref.sum() / div))
    refdx = (c[:, None].astype(np.float64) * wv[:, None] * g64) * float(inv_t)
    bar = gb * np.abs(c[:, None] * float(inv_t)) + 2.0 ** -22 * np.abs(refdx)
    assert lo.within(dx, refdx, bar)
  assert np.all(dx[~lo.valid(y)] == 0) and not np.any(np.signbit(dx[~lo.valid(y)]))
  if ndcg:
    nd, idcg = lo.ndcg32(pred, y, topn)
    assert np.array_equal(stats, lo.ndcg_stats(nd, idcg, wv, L))


@pytest.mark.parametrize("weights", ["none", "b", "b1"])
@pytest.mark.parametrize("red", list(REDS))
@pytest.mark.parametrize("mode", list(MODES))
def test_parity_every_loss_reduction_and_weighting(tfrs, mode, red, weights):
  pred, y, w = _data(37, 7, seed=1)
  y[0, 0] = -1; y[1, 3] = -1; y[2, 6] = -1          # padding at the front, middle and end
  w = None if weights == "none" else (w if weights == "b" else w[:, None])
  g = np.random.default_rng(2).uniform(-2, 2, size=37).astype(F32) if red == "none" else F32(1.5)
  _check(tfrs, MODES[mode], pred, y, w, REDS[red], g=g)


@pytest.mark.parametrize("L", [1, 2, 5, 31, 32, 33, 64, 255, 256, 1024])
@pytest.mark.parametrize("mode", list(MODES))
def test_list_lengths_and_cta_packing(tfrs, mode, L):
  W = lo.warps_per_cta(L)
  for B in (1, W + 1, 3 * W - 1) if L >= 255 else (1, W - 1 or 1, W, 5 * W + 3):
    pred, y, w = _data(B, L, seed=L + B)
    _check(tfrs, MODES[mode], pred, y, w, lo.RED_AUTO)


def test_large_batch_of_tutorial_lists(tfrs):
  pred, y, w = _data(8193, 5, seed=3)
  for mode in MODES.values():
    _check(tfrs, mode, pred, y, w, lo.RED_AUTO, ndcg=mode == lo.HINGE)


@pytest.mark.parametrize("mode", list(MODES))
def test_edge_inputs(tfrs, mode):
  m = MODES[mode]
  pred, y, w = _data(24, 40, seed=4)
  y[3] = -1                                  # a fully padded list
  y[4, :] = -1; y[4, 7] = 2                  # one valid item
  y[5] = 0                                   # no gain
  y[6, 1:] = -1                              # padding at the end
  y[7, :30] = np.nan                         # NaN labels are padding too
  _check(tfrs, m, pred, y, w, lo.RED_NONE, g=np.linspace(-1, 1, 24).astype(F32))
  ties, _, _ = _data(16, 64, seed=5)
  yt = np.ones((16, 64), F32); yt[:, ::7] = 2; yt[:, 5::11] = -1  # massive label ties
  _check(tfrs, m, ties, yt, None, lo.RED_SUM, seed=3, call=4)
  big, yb, wb = _data(16, 48, seed=6, scale=40.0, offset=1e5)     # +-1e5: the max-subtraction
  _check(tfrs, m, big, yb, wb, lo.RED_AUTO)
  _check(tfrs, m, pred, y, w, lo.RED_AUTO, T=0.37)                 # temperature
  _check(tfrs, m, pred, y, w, lo.RED_SUM, T=3.0, topn=3)
  _check(tfrs, m, pred, y, w, lo.RED_AUTO, topn=1000)              # topn larger than every list


def test_ndcg_topn_and_ideal_rankings(tfrs):
  ops = tfrs.ops
  y = np.float32([[3, 2, 0, -1], [0, 1, 2, 3], [0, 0, 0, 0]])
  pred = np.float32([[3, 2, 1, 9], [3, 2, 1, 0], [1, 2, 3, 4]])
  for topn in (None, 1, 2, 3, 10):
    stats, nd = ops.listwise_ndcg(torch.tensor(pred, device="cuda"), torch.tensor(y, device="cuda"), topn=topn, per_list=True)
    ref, idcg = lo.ndcg32(pred, y, topn)
    assert np.array_equal(nd.cpu().numpy(), ref)
    assert np.array_equal(stats.cpu().numpy(), lo.ndcg_stats(ref, idcg, None, 4))
  assert nd.cpu().numpy()[0] == 1.0


def test_determinism_and_garbage_workspace(tfrs):
  from recommenders_b200 import _ffi
  pred, y, w = _data(300, 33, seed=7, labels=2)
  pt, yt, wt = (torch.tensor(a, device="cuda") for a in (pred, y, w))

  def once(loss):
    p = pt.clone().requires_grad_(True)
    m = tfrs.metrics.NDCGMetric(topn=5)
    task = tfrs.tasks.Ranking(loss=loss, metrics=[m])
    out = task(yt, p, sample_weight=wt)
    out.backward()
    return out.detach().cpu().numpy().tobytes(), p.grad.cpu().numpy().tobytes(), m._acc.cpu().numpy().tobytes()

  for cls in (tfrs.losses.ListMLELoss, tfrs.losses.PairwiseHingeLoss, tfrs.losses.SoftmaxLoss):
    a = once(cls(seed=11) if cls is tfrs.losses.ListMLELoss else cls())
    for buf in _ffi._ws_cache.values():
      buf.fill_(0xA5)
    b = once(cls(seed=11) if cls is tfrs.losses.ListMLELoss else cls())
    assert a == b
  mle = tfrs.losses.ListMLELoss(seed=11)
  first = once(mle)
  assert once(mle)[1] != first[1]            # the next call shuffles the (many) label ties differently
  assert first == once(tfrs.losses.ListMLELoss(seed=11))


def test_ndcg_metric_update_state_equals_the_fused_value(tfrs):
  pred, y, w = _data(50, 9, seed=8)
  pt, yt, wt = (torch.tensor(a, device="cuda") for a in (pred, y, w))
  fused, alone, other = tfrs.metrics.NDCGMetric(topn=4), tfrs.metrics.NDCGMetric(topn=4), tfrs.metrics.NDCGMetric(name="n2")
  task = tfrs.tasks.Ranking(loss=tfrs.losses.SoftmaxLoss(), metrics=[fused, other])
  before = tfrs.ops.launch_count()
  task(yt, pt, sample_weight=wt)
  alone.update_state(yt, pt, sample_weight=wt)
  assert np.array_equal(fused._acc.cpu().numpy(), alone._acc.cpu().numpy())
  assert tfrs.ops.launch_count() - before == 3    # the loss with the fused NDCG, `other` (topn=None), `alone`
  nd, idcg = lo.ndcg32(pred, y, None)
  assert np.array_equal(other._acc.cpu().numpy(), lo.ndcg_stats(nd, idcg, w, 9))
  # any other loss: the metric updates itself through the metric-only launch
  mse_task = tfrs.tasks.Ranking(loss=tfrs.losses.MeanSquaredError(), metrics=[tfrs.metrics.NDCGMetric(topn=4)])
  mse_task(yt, pt)
  nd, idcg = lo.ndcg32(pred, y, 4)
  assert np.array_equal(mse_task.metrics[0]._acc.cpu().numpy(), lo.ndcg_stats(nd, idcg, None, 9))


def test_errors(tfrs):
  ops = tfrs.ops
  p = torch.zeros((4, 1025), device="cuda")
  with pytest.raises(ValueError):
    ops.listwise_loss(p, p, mode=ops.LIST_LOSS_SOFTMAX)
  p = torch.zeros((4, 6), device="cuda")
  with pytest.raises(NotImplementedError):
    tfrs.losses.SoftmaxLoss()(p, p, sample_weight=torch.ones((4, 6), device="cuda"))
  with pytest.raises(ValueError):
    tfrs.losses.SoftmaxLoss()(p, torch.zeros((4, 5), device="cuda"))
  out = tfrs.losses.PairwiseHingeLoss()(p[:, :, None], p[:, :, None])    # [B, L, 1] is squeezed
  assert out.shape == ()


# ------------------------------------------------------------------------------------------------
# the reference's listwise_ranking tutorial, restated on synthetic ratings
# ------------------------------------------------------------------------------------------------
def _ratings(n_users=60, n_movies=200, per_user=40, seed=0):
  rng = np.random.default_rng(seed)
  taste = rng.normal(size=(n_users, 4)); feat = rng.normal(size=(n_movies, 4))
  users, movies, ratings = [], [], []
  for u in range(n_users):
    for m in rng.choice(n_movies, size=per_user, replace=False):
      users.append(u); movies.append(m)
      ratings.append(float(np.clip(np.round(3 + 1.5 * taste[u] @ feat[m] / 2), 1, 5)))
  return np.array(users), np.array(movies), np.array(ratings, np.float32)


class _RankingModel(torch.nn.Module):
  def __init__(self, tfrs, loss, n_users, n_movies):
    super().__init__()
    self.model = tfrs.Model()
    self.user_embeddings = tfrs.layers.embedding.Embedding(n_users + 1, 32)
    self.movie_embeddings = tfrs.layers.embedding.Embedding(n_movies + 1, 32)
    self.score_model = torch.nn.Sequential(tfrs.layers.blocks.Dense(256, activation="relu"),
                                           tfrs.layers.blocks.Dense(64, activation="relu"), tfrs.layers.blocks.Dense(1))
    self.task = tfrs.tasks.Ranking(loss=loss, metrics=[tfrs.metrics.NDCGMetric(name="ndcg_metric"),
                                                       tfrs.metrics.RootMeanSquaredError()])

  def forward(self, features):
    u = self.user_embeddings(features["user_id"])
    m = self.movie_embeddings(features["movie_title"])
    B, L = features["movie_title"].shape
    x = torch.cat([u[:, None, :].expand(B, L, u.shape[1]), m], dim=2).reshape(B * L, -1)
    return self.score_model(x).reshape(B, L, 1)


def _tutorial_model(tfrs, loss, n_users, n_movies):
  core = _RankingModel(tfrs, loss, n_users, n_movies)

  class M(tfrs.Model):
    def __init__(self):
      super().__init__()
      self.core = core

    def compute_loss(self, features, training=False):
      labels = features["user_rating"]
      scores = self.core(features)
      return self.core.task(labels=labels, predictions=scores.squeeze(-1))
  return M()


def test_listwise_ranking_tutorial(tfrs):
  from recommenders_b200.examples import movielens
  users, movies, ratings = _ratings()
  ds = tfrs.data.Dataset.from_tensor_slices({"user_id": torch.tensor(users, device="cuda"),
                                            "movie_title": torch.tensor(movies, device="cuda"),
                                            "user_rating": torch.tensor(ratings, device="cuda")})
  train = movielens.sample_listwise(ds, 50, 5, seed=42)
  (el,) = list(train)
  assert tuple(el["movie_title"].shape) == (3000, 5)
  batches = list(train.batch(256))
  random_ndcg = tfrs.metrics.NDCGMetric()
  g = torch.Generator(device="cuda"); g.manual_seed(0)
  for b in batches:
    random_ndcg.update_state(b["user_rating"], torch.rand(b["user_rating"].shape, generator=g, device="cuda"))
  for loss in (tfrs.losses.MeanSquaredError(), tfrs.losses.PairwiseHingeLoss(), tfrs.losses.ListMLELoss()):
    torch.manual_seed(0)
    model = _tutorial_model(tfrs, loss, 60, 200)
    model.compile(optimizer=tfrs.optimizers.Adagrad(0.1))
    first = float(model.evaluate(batches)["loss"])
    hist = model.fit(batches, epochs=4)
    assert all(np.isfinite(float(h["loss"])) for h in hist)
    ev = model.evaluate(batches, return_dict=True)
    assert {"ndcg_metric", "root_mean_squared_error", "loss"} <= set(ev)
    assert float(ev["loss"]) < first, (type(loss).__name__, first, float(ev["loss"]))
    assert ev["ndcg_metric"] > random_ndcg.result() + 0.02, (type(loss).__name__, ev["ndcg_metric"], random_ndcg.result())
