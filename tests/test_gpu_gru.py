"""K19 on the H100: `ops.gru` and `layers.GRU` against the float64 oracle (tests/gru_oracle.py) over units, batch tiles,
lengths, input widths (both K6 routes), biases, initial states and masks; bitwise invariances; launch counts; input
checks; and the sequential retrieval tutorial's GRU query tower trained end to end."""
import math

import numpy as np
import pytest
import torch

import gru_oracle as go
import recommenders_b200 as tfrs
from recommenders_b200 import ops
from recommenders_b200.data import Dataset
from recommenders_b200.layers.embedding import Embedding

pytestmark = pytest.mark.gpu

SMEM_MAX = 227 * 1024


def _row_tile(u):
  """The batch rows of one CTA for u units (csrc/rnn.cuh rnn_tile)."""
  jt = 32
  while jt < u and jt < 256:
    jt *= 2
  uj = 1
  while uj * jt < u:
    uj *= 2
  return (256 // jt) * (8 // uj)


def _resident_edges(smem_bytes):
  """Every u after which the whole U (or U^T) stops or starts fitting in shared memory next to the step buffers
  (csrc/rnn.cuh rnn_smem); not monotonic in u, since the row tile halves as u passes a power of two."""
  return [u for u in range(1, ops.GRU_MAX_UNITS) if (smem_bytes(u) <= SMEM_MAX) != (smem_bytes(u + 1) <= SMEM_MAX)]


FWD_EDGES = _resident_edges(lambda u: 4 * (2 * _row_tile(u) * u + u * 3 * u))              # h buffers + U
BWD_EDGES = _resident_edges(lambda u: 4 * (2 * _row_tile(u) * 3 * u + 3 * u * (u + 1)))     # dgr buffers + U^T
UNITS = sorted({1, 2, 31, 32, 33, 64, 65, 127, 128, 129, 257, 512, 513, 600, 768, 769, 1024, 1025, ops.GRU_MAX_UNITS}
               | {e + d for e in FWD_EDGES + BWD_EDGES for d in (-1, 0, 1)})


def _cu(a, grad=False):
  return None if a is None else torch.from_numpy(np.ascontiguousarray(a)).cuda().requires_grad_(grad)


def _mask(kind, B, T, rng):
  if kind is None:
    return None
  if kind == "random":
    m = rng.rand(B, T) < 0.6
  elif kind == "leading":          # left padding: the first steps of each row are masked
    m = np.arange(T)[None] >= rng.randint(0, T + 1, size=(B, 1))
  elif kind == "trailing":         # right padding
    m = np.arange(T)[None] < rng.randint(0, T + 1, size=(B, 1))
  else:                            # "all": some rows entirely masked, the others random
    m = rng.rand(B, T) < 0.5
    m[::3] = False
  return m


def _inputs(B, T, D, u, bias, h0, seed):
  rng = np.random.RandomState(seed)
  x = rng.normal(size=(B, T, D)).astype(np.float32)
  W = (rng.uniform(-1, 1, size=(D, 3 * u)) * math.sqrt(6 / (D + 3 * u))).astype(np.float32)
  U = (rng.normal(size=(u, 3 * u)) / math.sqrt(u)).astype(np.float32)
  b = (rng.normal(size=(2, 3 * u)) * 0.1).astype(np.float32) if bias else None
  h = rng.uniform(-1, 1, size=(B, u)).astype(np.float32) if h0 else None
  return rng, x, W, U, b, h


def _check(name, got, exp):
  got = got.detach().double().cpu().numpy() if isinstance(got, torch.Tensor) else got
  scale = np.abs(exp).max() if exp.size else 0.0
  err = np.abs(got - exp).max() if exp.size else 0.0
  assert got.shape == exp.shape, (name, got.shape, exp.shape)
  assert err <= 1e-5 * scale, f"{name}: max |error| {err:.3g} > 1e-5 * max |value| {scale:.3g}"


def _run_case(B, T, D, u, bias=True, h0=True, mask=None, seq=None, seed=0, mask_dtype=torch.bool):
  rng, x, W, U, b, h = _inputs(B, T, D, u, bias, h0, seed)
  m = _mask(mask, B, T, rng)
  seq = m is None if seq is None else seq
  xt, Wt, Ut, bt, ht = _cu(x, True), _cu(W, True), _cu(U, True), _cu(b, True), _cu(h, True)
  mt = None if m is None else torch.from_numpy(m).cuda().to(mask_dtype)
  out, hT = ops.gru(xt, Wt, Ut, bt, ht, mt, return_sequences=seq)
  g_seq = rng.normal(size=(B, T, u)).astype(np.float32) if seq else None
  g_last = rng.normal(size=(B, u)).astype(np.float32)
  loss = (hT * _cu(g_last)).sum()
  if seq:
    loss = loss + (out * _cu(g_seq)).sum()
  loss.backward()
  eseq, ehT, _ = go.forward(x, W, U, b, h, m)
  g = go.backward(x, W, U, b, h, m, g_seq, g_last)
  if seq:
    _check("seq", out, eseq)
  _check("h_T", hT, ehT)
  _check("dx", xt.grad, g["dx"])
  _check("dW", Wt.grad, g["dW"])
  _check("dU", Ut.grad, g["dU"])
  if bias:
    _check("dbias", bt.grad, g["dbias"])
  if h0:
    _check("dh0", ht.grad, g["dh0"])


def test_the_resident_boundaries_are_where_the_plan_says():
  # U resident to u = 136; U^T resident to u = 123 and at u = 129, 130, where the row tile halves (DESIGN.md K19)
  assert FWD_EDGES == [136] and BWD_EDGES == [123, 128, 130]
  assert {122, 124, 127, 131, 135, 137} <= set(UNITS)


@pytest.mark.parametrize("u", UNITS)
def test_units_and_batch_tiles_match_the_oracle(u):
  R = _row_tile(u)
  for i, B in enumerate(sorted({1, R - 1, R + 1, 3 * R + 2} - {0})):
    _run_case(B, 10, 32, u, seed=u * 10 + i)
    _run_case(B, 10, 32, u, mask="random", seed=u * 10 + i + 5)


@pytest.mark.parametrize("T", [1, 2, 10, 64])
@pytest.mark.parametrize("D", [1, 3, 32, 300])
def test_lengths_and_input_widths_match_the_oracle(T, D):
  _run_case(65, T, D, 32, seed=T * 1000 + D)
  _run_case(65, T, D, 32, mask="random", seed=T * 1000 + D + 1)


def test_both_dense_routes_are_covered():
  assert not ops.dense_uses_tc(65 * 10, 32, 96)
  assert ops.dense_uses_tc(65 * 64, 300, 96)               # the projection of (T, D) = (64, 300) above
  assert ops.dense_uses_tc(200 * 10, 128, 384)             # dU of the case below
  _run_case(200, 10, 300, 128, seed=11)
  _run_case(200, 10, 300, 128, mask="random", seed=12)


@pytest.mark.parametrize("bias", [True, False])
@pytest.mark.parametrize("h0", [True, False])
@pytest.mark.parametrize("mask", [None, "random", "leading", "trailing", "all"])
def test_options_and_masks_match_the_oracle(bias, h0, mask):
  dtype = {None: torch.bool, "random": torch.bool, "leading": torch.int32, "trailing": torch.int64, "all": torch.int32}[mask]
  _run_case(40, 10, 3, 33, bias=bias, h0=h0, mask=mask, seed=3, mask_dtype=dtype)


def test_masked_steps_do_no_arithmetic():
  """A masked step carries h bit for bit: scattered masked steps give the final-state bits of the same kept steps moved
  to the front of the row (the masked ones after them), at the same [B, T]."""
  B, T, D, u = 70, 12, 16, 32
  rng, x, W, U, b, h = _inputs(B, T, D, u, True, True, 21)
  m = rng.rand(B, T) < 0.5
  order = np.argsort(~m, axis=1, kind="stable")           # kept steps first, in order, then the masked ones
  x2 = np.take_along_axis(x, order[:, :, None], 1)
  m2 = np.arange(T)[None] < m.sum(1, keepdims=True)
  with torch.no_grad():
    _, a = ops.gru(_cu(x), _cu(W), _cu(U), _cu(b), _cu(h), _cu(m))
    _, c = ops.gru(_cu(x2), _cu(W), _cu(U), _cu(b), _cu(h), _cu(m2))
  assert torch.equal(a, c)
  rows = ~m.any(1)
  if rows.any():
    assert torch.equal(a[torch.from_numpy(rows).cuda()], _cu(h)[torch.from_numpy(rows).cuda()])


def test_no_grad_and_grad_forwards_are_bitwise_equal():
  B, T, D, u = 90, 10, 32, 65
  _, x, W, U, b, h = _inputs(B, T, D, u, True, True, 5)
  with torch.no_grad():
    s0, h0 = ops.gru(_cu(x), _cu(W), _cu(U), _cu(b), _cu(h), return_sequences=True)
  s1, h1 = ops.gru(_cu(x, True), _cu(W, True), _cu(U, True), _cu(b, True), _cu(h, True), return_sequences=True)
  assert h1.requires_grad and torch.equal(s0, s1.detach()) and torch.equal(h0, h1.detach())


def test_two_identical_steps_are_bitwise_equal():
  B, T, D, u = 300, 20, 64, 128
  rng, x, W, U, b, h = _inputs(B, T, D, u, True, True, 9)
  m = _cu(rng.rand(B, T) < 0.8)
  g = _cu(rng.normal(size=(B, u)).astype(np.float32))

  def step():
    ts = [_cu(a, True) for a in (x, W, U, b, h)]
    _, hT = ops.gru(*ts, mask=m)
    (hT * g).sum().backward()
    return [hT.detach()] + [t.grad for t in ts]

  for a, c in zip(step(), step()):
    assert torch.equal(a, c)


@pytest.mark.parametrize("T", [1, 64])
def test_one_launch_each_way_beyond_the_dense_calls(T):
  B, D, u = 100, 32, 32
  _, x, W, U, b, h = _inputs(B, T, D, u, True, True, 2)
  xt, Wt, Ut, bt, ht = (_cu(a, True) for a in (x, W, U, b, h))

  # the K6 calls alone: the projection forward and backward, and dU / db_r as a Dense backward with no dx
  n = ops.launch_count()
  gx = ops.dense(xt.reshape(B * T, D), Wt, bt[0])
  k6_fwd = ops.launch_count() - n
  hp = torch.zeros((B * T, u), device="cuda")
  gr = ops.dense(hp, Ut, bt[1])
  n = ops.launch_count()
  (gx.sum() + gr.sum()).backward()
  k6_bwd = ops.launch_count() - n

  n = ops.launch_count()
  _, hT = ops.gru(xt, Wt, Ut, bt, ht)
  fwd = ops.launch_count() - n
  n = ops.launch_count()
  hT.sum().backward()
  bwd = ops.launch_count() - n
  assert fwd == k6_fwd + 1
  assert bwd == k6_bwd + 1


def test_the_layer_with_an_attached_mask_state_and_config():
  torch.manual_seed(0)
  B, T, n, d, u = 64, 10, 50, 16, 24
  rng = np.random.RandomState(4)
  ids = rng.randint(0, n, size=(B, T))
  ids[rng.rand(B, T) < 0.3] = 0
  emb = Embedding(n, d, mask_zero=True)
  layer = tfrs.layers.GRU(u, return_state=True)
  h0 = torch.from_numpy(rng.normal(size=(B, u)).astype(np.float32)).cuda()
  e = emb(torch.from_numpy(ids).cuda())
  out, state = layer(e, initial_state=[h0])
  assert torch.equal(out, state)
  args = [a.detach().cpu().numpy() for a in (e, layer.kernel, layer.recurrent_kernel, layer.bias, h0)]
  _, exp, _ = go.forward(*args, mask=ids != 0)
  _check("layer h_T", out, exp)
  assert layer.bias.shape == (2, 3 * u) and not layer.bias.detach().any()
  rk = layer.recurrent_kernel.detach().double()
  assert torch.allclose(rk @ rk.T, torch.eye(u, dtype=torch.float64, device="cuda"), atol=1e-5)
  with pytest.raises(NotImplementedError, match="return_sequences"):
    tfrs.layers.GRU(u, return_sequences=True)(e)
  seq = tfrs.layers.GRU(u, return_sequences=True)(torch.randn((3, 5, d), device="cuda"))
  assert seq.shape == (3, 5, u)


def test_input_checks():
  W, U = torch.zeros((4, 6), device="cuda"), torch.zeros((2, 6), device="cuda")
  with pytest.raises(ValueError, match="T = 0"):
    ops.gru(torch.zeros((3, 0, 4), device="cuda"), W, U)
  out, h = ops.gru(torch.zeros((0, 5, 4), device="cuda"), W, U, return_sequences=True)
  assert out.shape == (0, 5, 2) and h.shape == (0, 2)
  big = ops.GRU_MAX_UNITS + 1
  with pytest.raises(ValueError, match=str(ops.GRU_MAX_UNITS)):
    ops.gru(torch.zeros((1, 1, 4), device="cuda"), torch.zeros((4, 3 * big), device="cuda"),
            torch.zeros((big, 3 * big), device="cuda"))
  with pytest.raises(ValueError, match=str(ops.GRU_MAX_UNITS)):
    tfrs.layers.GRU(big)
  with pytest.raises(RuntimeError, match="CUDA"):
    ops.gru(torch.zeros((3, 5, 4)), W, U)
  with pytest.raises(RuntimeError, match="CUDA"):
    ops.gru(torch.zeros((3, 5, 4), device="cuda"), W, U, initial_state=torch.zeros((3, 2)))
  with pytest.raises(TypeError, match="gru: the mask"):
    ops.gru(torch.zeros((3, 5, 4), device="cuda"), W, U, mask=torch.ones((3, 5), device="cuda"))
  with pytest.raises(ValueError, match="gru: the mask has shape"):
    ops.gru(torch.zeros((3, 5, 4), device="cuda"), W, U, mask=torch.ones((3, 4), dtype=torch.bool, device="cuda"))
  with pytest.raises(NotImplementedError, match="return_sequences"):
    ops.gru(torch.zeros((3, 5, 4), device="cuda"), W, U, mask=torch.ones((3, 5), dtype=torch.bool, device="cuda"),
            return_sequences=True)
  for kw in ({"activation": "relu"}, {"reset_after": False}, {"dropout": 0.5}, {"recurrent_dropout": 0.5},
             {"go_backwards": True}, {"stateful": True}, {"time_major": True}):
    with pytest.raises(NotImplementedError, match=next(iter(kw))):
      tfrs.layers.GRU(4, **kw)


# ---- the sequential retrieval tutorial (docs/examples/sequential_retrieval.ipynb) on synthetic histories ----------------
TUTORIAL_TOP10_FLOOR = 0.45  # half the held-out top-10 accuracy this seeded run reached on an H100 (0.897)


def _histories(seed=0, n=300, rows=51200, T=10):
  """Seeded watch histories: a Markov chain over n string ids in which each id has three likely successors."""
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


class _SequentialModel(tfrs.Model):
  def __init__(self, query_model, candidate_model, task):
    super().__init__()
    self._query_model, self._candidate_model, self._task = query_model, candidate_model, task

  def compute_loss(self, features, training=False):
    query_embedding = self._query_model(features["context_movie_id"])
    candidate_embedding = self._candidate_model(features["label_movie_id"])
    return self._task(query_embedding, candidate_embedding, compute_metrics=not training)


def test_sequential_retrieval_tutorial_trains_end_to_end(monkeypatch):
  def no_rnn(*a, **k):
    raise AssertionError("a torch / cuDNN RNN op ran")

  for mod in (torch, torch._VF):
    for name in ("gru", "gru_cell", "rnn_tanh", "rnn_relu", "lstm", "_cudnn_rnn"):
      if hasattr(mod, name):
        monkeypatch.setattr(mod, name, no_rnn)
  for cls in (torch.nn.GRU, torch.nn.GRUCell, torch.nn.RNN, torch.nn.LSTM):
    monkeypatch.setattr(cls, "forward", no_rnn)

  ids, ctx, label = _histories()
  n_train = 49152
  torch.manual_seed(0)
  query_model = torch.nn.Sequential(tfrs.layers.StringLookup(vocabulary=ids, mask_token=None),
                                    Embedding(len(ids) + 1, 32), tfrs.layers.GRU(32))
  candidate_model = torch.nn.Sequential(tfrs.layers.StringLookup(vocabulary=ids, mask_token=None),
                                        Embedding(len(ids) + 1, 32))
  movies = Dataset.from_tensor_slices(ids)
  task = tfrs.tasks.Retrieval(metrics=tfrs.metrics.FactorizedTopK(candidates=movies.batch(128).map(candidate_model)))
  model = _SequentialModel(query_model, candidate_model, task)
  model.compile(optimizer=tfrs.optimizers.Adagrad(learning_rate=0.1))
  train = Dataset.from_tensor_slices({"context_movie_id": ctx[:n_train], "label_movie_id": label[:n_train]}).batch(1024)
  test = Dataset.from_tensor_slices({"context_movie_id": ctx[n_train:], "label_movie_id": label[n_train:]}).batch(2560)

  before = model.evaluate(test)
  gru = query_model[2]
  w0 = gru.recurrent_kernel.detach().clone()
  hist = model.fit(train, epochs=3)
  after = model.evaluate(test)
  top10 = float(after["factorized_top_k/top_10_categorical_accuracy"])
  print(f"sequential tutorial: loss {float(before['loss']):.4f} -> {float(after['loss']):.4f}, "
        f"held-out top-10 accuracy {float(before['factorized_top_k/top_10_categorical_accuracy']):.4f} -> {top10:.4f}")
  assert all(np.isfinite(float(h["loss"])) for h in hist)
  assert float(after["loss"]) < float(before["loss"])
  assert top10 >= TUTORIAL_TOP10_FLOOR
  # the GRU's weights are ordinary dense parameters: Adagrad moved them
  assert not torch.equal(w0, gru.recurrent_kernel.detach())
