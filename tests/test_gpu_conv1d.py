"""K27 on the H100: `ops.conv1d` and `layers.Conv1D` against the float64 oracle (tests/conv1d_oracle.py) per element, with
the bar of the split-GEMM edge tests, on both routes, across tile, chunk and width edges, sequence ends and batch-row
boundaries, every activation and use_bias=False; bitwise invariances; launch counts; and a NextItNet-style query tower
trained end to end on the sequential-retrieval synthetic histories with torch's convolutions disabled."""
import numpy as np
import pytest
import torch

import conv1d_oracle as co
import recommenders_b200 as tfrs
from recommenders_b200 import ops
from recommenders_b200.data import Dataset
from recommenders_b200.layers.embedding import Embedding
from recommenders_b200.layers.feature_interaction.dcn import _ACTIVATIONS

pytestmark = pytest.mark.gpu

FUSED = (None, "linear", "relu", "sigmoid")
LIPSCHITZ = 1.2   # max |act'| of every activation in dcn._ACTIVATIONS (gelu's is 1.13)


def _cu(a, grad=False):
  return None if a is None else torch.from_numpy(np.ascontiguousarray(a)).cuda().requires_grad_(grad)


def _f64(t):
  return t.detach().double().cpu().numpy()


def _E(name, got, ref, tol):
  got = _f64(got) if isinstance(got, torch.Tensor) else got
  assert got.shape == ref.shape, (name, got.shape, ref.shape)
  assert np.isfinite(got).all(), f"{name}: non-finite results"
  err = np.abs(got - ref)
  bad = err > tol
  if bad.any():
    i = tuple(np.argwhere(bad)[0])
    raise AssertionError(f"{name}: {int(bad.sum())} elements miss the bar; first {i}: got {got[i]!r} ref {ref[i]!r} "
                         f"err {err[i]:.3e} bar {tol[i]:.3e}")


def _run(B, T, C, k, F, s=1, d=1, padding="valid", act=None, bias=True, seed=0, tc=None):
  """One forward and backward of ops.conv1d (a callable activation applied to the fused linear output, as Conv1D does),
  every output and gradient checked per element against the float64 oracle."""
  rng = np.random.RandomState(seed)
  x = rng.normal(size=(B, T, C)).astype(np.float32)
  W = (rng.normal(size=(k, C, F)) / np.sqrt(k * C)).astype(np.float32)
  b = (rng.normal(size=F) * 0.5).astype(np.float32) if bias else None
  T_out, p, _ = co.geometry(T, k, s, d, padding)
  if tc is not None:
    assert ops.conv1d_uses_tc(B, T_out, C, k, F) == tc
  xt, Wt, bt = _cu(x, True), _cu(W, True), _cu(b, True)
  fused = act in FUSED
  y = ops.conv1d(xt, Wt, bt, s, padding, d, activation=act if fused else None)
  if not fused:
    y = _ACTIVATIONS[act](y)
  g = rng.normal(size=(B, T_out, F)).astype(np.float32)
  y.backward(_cu(g))

  z64, y64, col = co.forward(x, W, b, s, d, padding, act)
  W2 = W.astype(np.float64).reshape(k * C, F)
  amax_x = float(np.abs(x).max())
  zbar = co.ebar(col, W2, amax_a=amax_x).reshape(B, T_out, F)
  if b is not None:
    zbar = zbar + 2.0 ** -22 * np.abs(b.astype(np.float64))
  ybar = zbar if act in (None, "linear") else LIPSCHITZ * zbar + 2.0 ** -20 * np.abs(y64) + 2.0 ** -22 * np.abs(z64)
  _E("y", y, y64, ybar)

  # dz as the kernels form it: from the saved output for a fused activation, torch's fp32 gradient of a callable one
  yg = _f64(y)
  if act in (None, "linear"):
    dz = g.astype(np.float64)
  elif act == "relu":
    dz = g * (yg > 0)
  elif act == "sigmoid":
    dz = g * yg * (1 - yg)
  else:
    with torch.no_grad():
      z = ops.conv1d(xt, Wt, bt, s, padding, d)
    z.requires_grad_()
    dz = _f64(torch.autograd.grad(_ACTIVATIONS[act](z), z, _cu(g))[0])
  dx64, dW64, db64 = co.backward(x, W, dz, s, d, padding)
  dz2 = dz.reshape(B * T_out, F)
  _E("dx", xt.grad, dx64, co.col2im(co.ebar(dz2, W2.T), B, T, C, k, s, d, p, T_out))
  _E("dW", Wt.grad, dW64, co.ebar(col.T, dz2, amax_a=amax_x).reshape(k, C, F))
  if bias:
    _E("dbias", bt.grad, db64, 1e-5 * np.abs(dz2).sum(0))


# ---- both routes, every padding, stride and dilation ---------------------------------------------------------------------
GEOMETRIES = [(p, s, d) for p in co.PADDINGS for s, d in ((1, 1), (2, 1), (3, 1), (1, 2), (1, 4))]


@pytest.mark.parametrize("padding,s,d", GEOMETRIES)
def test_cuda_core_route_every_geometry(padding, s, d):
  _run(5, 11, 6, 3, 7, s, d, padding, seed=s * 10 + d, tc=False)
  _run(3, 20, 70, 5, 65, s, d, padding, seed=s * 10 + d + 1, tc=False)    # M < 1024


@pytest.mark.parametrize("padding,s,d", GEOMETRIES)
def test_tensor_core_route_every_geometry(padding, s, d):
  _run(96, 40, 32, 3, 64, s, d, padding, seed=s * 10 + d + 2, tc=True)


# ---- tile, chunk and width edges ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("B", [1023, 1024, 1025, 1151, 1152, 1153, 2047, 2048, 2049])
def test_rows_across_tile_and_chunk_edges(B):
  """M = B T_out across the 128-row tiles and, for dW, the 1024-step chunks of the reduction over B T_out."""
  _run(B, 1, 32, 3, 64, padding="causal", seed=B, tc=B >= 1024)


@pytest.mark.parametrize("B,T", [(127, 9), (128, 9), (129, 9), (57, 19)])
def test_rows_of_several_steps_across_tile_edges(B, T):
  _run(B, T, 64, 2, 96, padding="same", seed=B * T, tc=True)


@pytest.mark.parametrize("k,C", [(1, 1023), (1, 1024), (1, 1025), (2, 512), (3, 342), (4, 256), (5, 205), (17, 64)])
def test_reduction_width_across_the_chunk_edge(k, C):
  """K = k C across 1024: one accumulation chain at or below it, fixed-order chunks above."""
  _run(20, 60, C, k, 64, padding="causal", seed=k * 10000 + C, tc=True)


@pytest.mark.parametrize("F", [1, 17, 63, 65, 127, 129, 193])
def test_odd_filter_counts(F):
  _run(40, 30, 32, 3, F, padding="same", seed=F, tc=F >= 64)
  _run(7, 12, 10, 3, F, padding="valid", seed=F + 1, tc=False)


# ---- sequence ends ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("tc", [False, True])
def test_valid_minimum_and_single_steps(tc):
  B = 1100 if tc else 9
  for k, d in ((3, 1), (3, 2), (5, 4)):
    _run(B, d * (k - 1) + 1, 32, k, 64, d=d, padding="valid", seed=k + d, tc=tc)        # T_out = 1
  for padding in ("same", "causal"):
    for k, d in ((3, 1), (5, 2)):
      _run(B, 1, 32, k, 64, d=d, padding=padding, seed=k * d, tc=tc)                    # T = 1


@pytest.mark.parametrize("tc", [False, True])
def test_windows_crossing_both_ends_and_batch_rows(tc):
  """Short sequences under wide receptive fields: windows reach past both ends of every row, where a read into the
  neighbouring batch row would add a term far above the bar."""
  B = 400 if tc else 6
  for padding, k, d, T in (("same", 5, 2, 4), ("same", 7, 1, 3), ("causal", 3, 4, 5), ("same", 4, 3, 6)):
    _run(B, T, 64, k, 64, d=d, padding=padding, seed=k * 100 + T, tc=tc)
  _run(B, 7, 64, 4, 64, s=3, padding="same", seed=77, tc=tc)


# ---- activations and bias ---------------------------------------------------------------------------------------------
ACTS = [None, "linear", "relu", "sigmoid", "tanh", "swish", "silu", "gelu"]


@pytest.mark.parametrize("act", ACTS)
@pytest.mark.parametrize("bias", [True, False])
@pytest.mark.parametrize("tc", [False, True])
def test_every_activation_with_and_without_bias(act, bias, tc):
  B = 64 if tc else 4
  _run(B, 20, 32, 3, 64 if tc else 24, d=2, padding="causal", act=act, bias=bias, seed=ACTS.index(act), tc=tc)


def test_the_layer_matches_the_oracle_and_refuses_an_attached_mask():
  torch.manual_seed(0)
  layer = tfrs.layers.Conv1D(40, 3, padding="same", activation="tanh")
  x = np.random.RandomState(1).normal(size=(8, 12, 16)).astype(np.float32)
  y = layer(_cu(x))
  assert layer.kernel.shape == (3, 16, 40) and layer.bias.shape == (40,) and not layer.bias.detach().any()
  limit = np.sqrt(6.0 / (3 * 16 + 3 * 40))            # glorot_uniform with Keras's fans of a [3, 16, 40] kernel
  assert float(layer.kernel.detach().abs().max()) <= limit and float(layer.kernel.detach().abs().max()) > 0.9 * limit
  _, exp, _ = co.forward(x, _f64(layer.kernel), _f64(layer.bias), 1, 1, "same", "tanh")
  assert np.abs(_f64(y) - exp).max() <= 1e-5 * np.abs(exp).max()
  ids = torch.from_numpy(np.random.RandomState(2).randint(0, 5, size=(8, 12))).cuda()
  e = Embedding(5, 16, mask_zero=True)(ids)
  with pytest.raises(TypeError, match="does not support masking"):
    layer(e)
  assert layer(Embedding(5, 16)(ids)).shape == (8, 12, 40)


def test_input_checks():
  W = torch.zeros((3, 4, 5), device="cuda")
  with pytest.raises(RuntimeError, match="CUDA"):
    ops.conv1d(torch.zeros((2, 5, 4)), W)
  with pytest.raises(ValueError, match="kernel"):
    ops.conv1d(torch.zeros((2, 5, 3), device="cuda"), W)
  with pytest.raises(ValueError, match="zero or negative"):
    ops.conv1d(torch.zeros((2, 2, 4), device="cuda"), W)
  with pytest.raises(ValueError, match="not fused"):
    ops.conv1d(torch.zeros((2, 5, 4), device="cuda"), W, activation="tanh")
  y = ops.conv1d(torch.zeros((0, 5, 4), device="cuda", requires_grad=True), W, padding="same")
  assert y.shape == (0, 5, 5)


# ---- reproducibility and launches --------------------------------------------------------------------------------------
def _inputs(B, T, C, k, F, seed):
  rng = np.random.RandomState(seed)
  return (rng.normal(size=(B, T, C)).astype(np.float32), (rng.normal(size=(k, C, F)) / np.sqrt(k * C)).astype(np.float32),
          rng.normal(size=F).astype(np.float32), rng)


@pytest.mark.parametrize("shape", [(6, 20, 8, 3, 24), (64, 40, 64, 3, 64), (40, 60, 400, 3, 96)])
def test_no_grad_and_grad_forwards_are_bitwise_equal(shape):
  x, W, b, _ = _inputs(*shape, 3)
  for act in ("relu", "sigmoid"):
    with torch.no_grad():
      y0 = ops.conv1d(_cu(x), _cu(W), _cu(b), 1, "causal", 2, activation=act)
    y1 = ops.conv1d(_cu(x, True), _cu(W, True), _cu(b, True), 1, "causal", 2, activation=act)
    assert y1.requires_grad and torch.equal(y0, y1.detach())


@pytest.mark.parametrize("shape", [(6, 20, 8, 3, 24), (64, 40, 64, 3, 64), (40, 60, 400, 3, 96)])
def test_two_identical_steps_are_bitwise_equal(shape):
  x, W, b, rng = _inputs(*shape, 4)
  g = _cu(rng.normal(size=(shape[0], shape[1], shape[4])).astype(np.float32))

  def step():
    ts = [_cu(a, True) for a in (x, W, b)]
    y = ops.conv1d(*ts, 1, "same", 1, activation="relu")
    y.backward(g)
    return [y.detach()] + [t.grad for t in ts]

  for a, c in zip(step(), step()):
    assert torch.equal(a, c)


@pytest.mark.parametrize("shape,tc", [((6, 20, 8, 3, 24), False), ((64, 40, 64, 3, 64), True), ((40, 60, 400, 3, 96), True)])
def test_launches_each_way(shape, tc):
  """The tensor-core route is K6's launches with the window gather in place of the A image; the CUDA-core route adds
  the im2col gather each way; both add one col2im launch backward."""
  B, T, C, k, F = shape
  assert ops.conv1d_uses_tc(B, T, C, k, F) == tc
  x, W, b, rng = _inputs(B, T, C, k, F, 5)
  col = torch.zeros((B * T, k * C), device="cuda", requires_grad=True)
  W2, b2 = _cu(W.reshape(k * C, F), True), _cu(b, True)
  n = ops.launch_count()
  z = ops.dense(col, W2, b2)
  k6_fwd = ops.launch_count() - n
  n = ops.launch_count()
  z.sum().backward()
  k6_bwd = ops.launch_count() - n

  ts = [_cu(a, True) for a in (x, W, b)]
  n = ops.launch_count()
  y = ops.conv1d(*ts, 1, "causal", 1)
  fwd = ops.launch_count() - n
  n = ops.launch_count()
  y.sum().backward()
  bwd = ops.launch_count() - n
  assert fwd == k6_fwd + (0 if tc else 1)
  assert bwd == k6_bwd + (1 if tc else 2)


# ---- a NextItNet-style query tower on the sequential retrieval tutorial's synthetic histories ---------------------------
TUTORIAL_TOP10_FLOOR = 0.45  # half the held-out top-10 accuracy this seeded run reached on an H100 (0.901)


def _histories(seed=0, n=300, rows=51200, T=10):
  """Seeded watch histories: a Markov chain over n string ids in which each id has three likely successors (as
  tests/test_gpu_gru.py)."""
  rng = np.random.RandomState(seed)
  succ = rng.randint(0, n, size=(n, 3))
  s = np.empty((rows, T + 1), np.int64)
  s[:, 0] = rng.randint(0, n, size=rows)
  for t in range(1, T + 1):
    nxt = succ[s[:, t - 1], rng.choice(3, p=[0.6, 0.25, 0.15], size=rows)]
    jump = rng.rand(rows) < 0.1
    s[:, t] = np.where(jump, rng.randint(0, n, size=rows), nxt)
  ids = np.array([str(1000 + i) for i in range(n)])
  return ids, ids[s[:, :T]], ids[s[:, T]]


class _ResidualConvs(torch.nn.Module):
  """[Conv1D(causal, dilation 1, 2, 4) + residual] x 2, then the last step."""

  def __init__(self, d):
    super().__init__()
    self.convs = torch.nn.ModuleList([tfrs.layers.Conv1D(d, 3, padding="causal", dilation_rate=r, activation="relu")
                                      for _ in range(2) for r in (1, 2, 4)])

  def forward(self, h):
    for conv in self.convs:
      h = h + conv(h)
    return h[:, -1, :]


class _SequentialModel(tfrs.Model):
  def __init__(self, query_model, candidate_model, task):
    super().__init__()
    self._query_model, self._candidate_model, self._task = query_model, candidate_model, task

  def compute_loss(self, features, training=False):
    query_embedding = self._query_model(features["context_movie_id"])
    candidate_embedding = self._candidate_model(features["label_movie_id"])
    return self._task(query_embedding, candidate_embedding, compute_metrics=not training)


def test_nextitnet_tower_trains_end_to_end(monkeypatch):
  def no_conv(*a, **k):
    raise AssertionError("a torch / cuDNN convolution ran")

  for mod in (torch, torch.nn.functional):
    for name in dir(mod):
      if name.startswith("conv") and callable(getattr(mod, name)):
        monkeypatch.setattr(mod, name, no_conv)
  for cls in (torch.nn.Conv1d, torch.nn.Conv2d):
    monkeypatch.setattr(cls, "forward", no_conv)

  ids, ctx, label = _histories()
  n_train = 49152
  torch.manual_seed(0)
  query_model = torch.nn.Sequential(tfrs.layers.StringLookup(vocabulary=ids, mask_token=None),
                                    Embedding(len(ids) + 1, 32), _ResidualConvs(32))
  candidate_model = torch.nn.Sequential(tfrs.layers.StringLookup(vocabulary=ids, mask_token=None),
                                        Embedding(len(ids) + 1, 32))
  movies = Dataset.from_tensor_slices(ids)
  task = tfrs.tasks.Retrieval(metrics=tfrs.metrics.FactorizedTopK(candidates=movies.batch(128).map(candidate_model)))
  model = _SequentialModel(query_model, candidate_model, task)
  model.compile(optimizer=tfrs.optimizers.Adagrad(learning_rate=0.1))
  train = Dataset.from_tensor_slices({"context_movie_id": ctx[:n_train], "label_movie_id": label[:n_train]}).batch(1024)
  test = Dataset.from_tensor_slices({"context_movie_id": ctx[n_train:], "label_movie_id": label[n_train:]}).batch(2560)

  before = model.evaluate(test)
  conv = query_model[2].convs[0]
  w0 = conv.kernel.detach().clone()
  hist = model.fit(train, epochs=3)
  after = model.evaluate(test)
  top10 = float(after["factorized_top_k/top_10_categorical_accuracy"])
  print(f"NextItNet tower: loss {float(before['loss']):.4f} -> {float(after['loss']):.4f}, "
        f"held-out top-10 accuracy {float(before['factorized_top_k/top_10_categorical_accuracy']):.4f} -> {top10:.4f}")
  assert all(np.isfinite(float(h["loss"])) for h in hist)
  assert float(after["loss"]) < float(before["loss"])
  assert top10 >= TUTORIAL_TOP10_FLOOR
  assert not torch.equal(w0, conv.kernel.detach())
