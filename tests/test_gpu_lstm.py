"""K20 on the H100: `ops.lstm` and `layers.LSTM` against the float64 oracle (tests/lstm_oracle.py) over units (with the
resident / streamed U boundaries), batch tiles, lengths, input widths (both K6 routes), biases, initial states and
masks; bitwise invariances; launch counts; the layer and its input checks; and the sequential retrieval tutorial with an
LSTM query tower trained end to end."""
import math

import numpy as np
import pytest
import torch

import lstm_oracle as lo
import recommenders_b200 as tfrs
from recommenders_b200 import ops
from recommenders_b200.data import Dataset
from recommenders_b200.layers.embedding import Embedding
from test_gpu_gru import _SequentialModel, _check, _cu, _histories, _mask, _resident_edges, _row_tile

pytestmark = pytest.mark.gpu

(FWD_RESIDENT,) = _resident_edges(lambda u: 4 * (2 * _row_tile(u) * u + u * 4 * u))              # h buffers + U
(BWD_RESIDENT,) = _resident_edges(lambda u: 4 * (2 * _row_tile(u) * 4 * u + 4 * u * (u + 1)))     # dz buffers + U^T
UNITS = sorted({1, 2, 31, 32, 33, 64, 65, 127, 128, 129, 257, 512, 513, 600, 768, 769, 1024, 1025, ops.LSTM_MAX_UNITS,
                FWD_RESIDENT - 1, FWD_RESIDENT, FWD_RESIDENT + 1, BWD_RESIDENT - 1, BWD_RESIDENT, BWD_RESIDENT + 1})


def _inputs(B, T, D, u, bias, state, seed):
  rng = np.random.RandomState(seed)
  x = rng.normal(size=(B, T, D)).astype(np.float32)
  W = (rng.uniform(-1, 1, size=(D, 4 * u)) * math.sqrt(6 / (D + 4 * u))).astype(np.float32)
  U = (rng.normal(size=(u, 4 * u)) / math.sqrt(u)).astype(np.float32)
  b = (rng.normal(size=4 * u) * 0.1).astype(np.float32) if bias else None
  h = rng.uniform(-1, 1, size=(B, u)).astype(np.float32) if state else None
  c = rng.uniform(-2, 2, size=(B, u)).astype(np.float32) if state else None
  return rng, x, W, U, b, h, c


def _run_case(B, T, D, u, bias=True, state=True, mask=None, seq=None, seed=0, mask_dtype=torch.bool, c_grad=True):
  rng, x, W, U, b, h, c = _inputs(B, T, D, u, bias, state, seed)
  m = _mask(mask, B, T, rng)
  seq = m is None if seq is None else seq
  xt, Wt, Ut, bt, ht, ct = (_cu(a, True) for a in (x, W, U, b, h, c))
  mt = None if m is None else torch.from_numpy(m).cuda().to(mask_dtype)
  out, hT, cT = ops.lstm(xt, Wt, Ut, bt, None if h is None else (ht, ct), mt, return_sequences=seq)
  g_seq = rng.normal(size=(B, T, u)).astype(np.float32) if seq else None
  g_h = rng.normal(size=(B, u)).astype(np.float32)
  g_c = rng.normal(size=(B, u)).astype(np.float32) if c_grad else None
  loss = (hT * _cu(g_h)).sum()
  if seq:
    loss = loss + (out * _cu(g_seq)).sum()
  if c_grad:
    loss = loss + (cT * _cu(g_c)).sum()
  loss.backward()
  eseq, ehT, ecT, _ = lo.forward(x, W, U, b, h, c, m)
  g = lo.backward(x, W, U, b, h, c, m, g_seq, g_h, g_c)
  if seq:
    _check("seq", out, eseq)
  _check("h_T", hT, ehT)
  _check("c_T", cT, ecT)
  _check("dx", xt.grad, g["dx"])
  _check("dW", Wt.grad, g["dW"])
  _check("dU", Ut.grad, g["dU"])
  if bias:
    _check("db", bt.grad, g["dbias"])
  if state:
    _check("dh0", ht.grad, g["dh0"])
    _check("dc0", ct.grad, g["dc0"])


def test_the_resident_boundaries_are_where_the_plan_says():
  assert 64 < BWD_RESIDENT < FWD_RESIDENT < 257
  assert FWD_RESIDENT + 1 in UNITS and BWD_RESIDENT - 1 in UNITS


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
  assert not ops.dense_uses_tc(65 * 10, 32, 128)
  assert ops.dense_uses_tc(65 * 64, 300, 128)              # the projection of (T, D) = (64, 300) above
  assert ops.dense_uses_tc(200 * 10, 128, 512)             # dU of the case below
  _run_case(200, 10, 300, 128, seed=11)
  _run_case(200, 10, 300, 128, mask="random", seed=12)


@pytest.mark.parametrize("bias", [True, False])
@pytest.mark.parametrize("state", [True, False])
@pytest.mark.parametrize("mask", [None, "random", "leading", "trailing", "all"])
def test_options_and_masks_match_the_oracle(bias, state, mask):
  dtype = {None: torch.bool, "random": torch.bool, "leading": torch.int32, "trailing": torch.int64, "all": torch.int32}[mask]
  _run_case(40, 10, 3, 33, bias=bias, state=state, mask=mask, seed=3, mask_dtype=dtype)


def test_gradients_from_h_alone_match_the_oracle():
  _run_case(70, 12, 16, 48, mask="random", seed=13, c_grad=False)
  _run_case(70, 12, 16, 48, seq=True, seed=14, c_grad=False)


def test_masked_steps_do_no_arithmetic():
  """A masked step carries h and c bit for bit: scattered masked steps give the final-state bits of the same kept steps
  moved to the front of the row (the masked ones after them), at the same [B, T]."""
  B, T, D, u = 70, 12, 16, 32
  rng, x, W, U, b, h, c = _inputs(B, T, D, u, True, True, 21)
  m = rng.rand(B, T) < 0.5
  order = np.argsort(~m, axis=1, kind="stable")           # kept steps first, in order, then the masked ones
  x2 = np.take_along_axis(x, order[:, :, None], 1)
  m2 = np.arange(T)[None] < m.sum(1, keepdims=True)
  with torch.no_grad():
    _, ha, ca = ops.lstm(_cu(x), _cu(W), _cu(U), _cu(b), (_cu(h), _cu(c)), _cu(m))
    _, hb, cb = ops.lstm(_cu(x2), _cu(W), _cu(U), _cu(b), (_cu(h), _cu(c)), _cu(m2))
  assert torch.equal(ha, hb) and torch.equal(ca, cb)
  rows = torch.from_numpy(~m.any(1)).cuda()
  if rows.any():
    assert torch.equal(ha[rows], _cu(h)[rows]) and torch.equal(ca[rows], _cu(c)[rows])


def test_no_grad_and_grad_forwards_are_bitwise_equal():
  B, T, D, u = 90, 10, 32, 65
  _, x, W, U, b, h, c = _inputs(B, T, D, u, True, True, 5)
  with torch.no_grad():
    s0, h0, c0 = ops.lstm(_cu(x), _cu(W), _cu(U), _cu(b), (_cu(h), _cu(c)), return_sequences=True)
  s1, h1, c1 = ops.lstm(_cu(x, True), _cu(W, True), _cu(U, True), _cu(b, True), (_cu(h, True), _cu(c, True)),
                        return_sequences=True)
  assert h1.requires_grad and c1.requires_grad
  assert torch.equal(s0, s1.detach()) and torch.equal(h0, h1.detach()) and torch.equal(c0, c1.detach())


def test_two_identical_steps_are_bitwise_equal():
  B, T, D, u = 300, 20, 64, 128
  rng, x, W, U, b, h, c = _inputs(B, T, D, u, True, True, 9)
  m = _cu(rng.rand(B, T) < 0.8)
  gh = _cu(rng.normal(size=(B, u)).astype(np.float32))
  gc = _cu(rng.normal(size=(B, u)).astype(np.float32))

  def step():
    ts = [_cu(a, True) for a in (x, W, U, b, h, c)]
    _, hT, cT = ops.lstm(*ts[:4], (ts[4], ts[5]), mask=m)
    ((hT * gh).sum() + (cT * gc).sum()).backward()
    return [hT.detach(), cT.detach()] + [t.grad for t in ts]

  for a, e in zip(step(), step()):
    assert torch.equal(a, e)


@pytest.mark.parametrize("T", [1, 64])
def test_one_launch_each_way_beyond_the_dense_calls(T):
  B, D, u = 100, 32, 32
  _, x, W, U, b, h, c = _inputs(B, T, D, u, True, True, 2)
  xt, Wt, Ut, bt, ht, ct = (_cu(a, True) for a in (x, W, U, b, h, c))

  # the K6 calls alone: the projection forward and backward, and dU as a Dense backward with no dx and no bias
  n = ops.launch_count()
  gx = ops.dense(xt.reshape(B * T, D), Wt, bt)
  k6_fwd = ops.launch_count() - n
  hp = torch.zeros((B * T, u), device="cuda")
  gr = ops.dense(hp, Ut)
  n = ops.launch_count()
  (gx.sum() + gr.sum()).backward()
  k6_bwd = ops.launch_count() - n

  n = ops.launch_count()
  _, hT, cT = ops.lstm(xt, Wt, Ut, bt, (ht, ct))
  fwd = ops.launch_count() - n
  n = ops.launch_count()
  (hT.sum() + cT.sum()).backward()
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
  layer = tfrs.layers.LSTM(u, return_state=True)
  h0 = torch.from_numpy(rng.normal(size=(B, u)).astype(np.float32)).cuda()
  c0 = torch.from_numpy(rng.normal(size=(B, u)).astype(np.float32)).cuda()
  e = emb(torch.from_numpy(ids).cuda())
  res = layer(e, initial_state=[h0, c0])
  assert isinstance(res, list) and len(res) == 3
  out, hT, cT = res
  assert torch.equal(out, hT) and cT.shape == (B, u)
  args = [a.detach().cpu().numpy() for a in (e, layer.kernel, layer.recurrent_kernel, layer.bias, h0, c0)]
  _, eh, ec, _ = lo.forward(*args, mask=ids != 0)
  _check("layer h_T", hT, eh)
  _check("layer c_T", cT, ec)
  bias = layer.bias.detach()
  assert bias.shape == (4 * u,) and torch.equal(bias[u:2 * u], torch.ones(u, device="cuda"))
  assert not bias[:u].any() and not bias[2 * u:].any()
  rk = layer.recurrent_kernel.detach().double()
  assert torch.allclose(rk @ rk.T, torch.eye(u, dtype=torch.float64, device="cuda"), atol=1e-5)
  with pytest.raises(NotImplementedError, match="return_sequences"):
    tfrs.layers.LSTM(u, return_sequences=True)(e)
  with pytest.raises(ValueError, match="two initial states"):
    layer(e, initial_state=[h0])
  seq = tfrs.layers.LSTM(u, return_sequences=True)(torch.randn((3, 5, d), device="cuda"))
  assert seq.shape == (3, 5, u)


def test_a_state_dict_round_trip_reproduces_the_outputs():
  torch.manual_seed(1)
  x = torch.randn((37, 9, 12), device="cuda")
  m = torch.rand((37, 9), device="cuda") < 0.7
  a = tfrs.layers.LSTM(20, return_state=True)
  with torch.no_grad():
    ra = a(x, mask=m)
  b = tfrs.layers.LSTM(20, return_state=True, kernel_initializer="zeros", recurrent_initializer="zeros")
  with torch.no_grad():
    b(x, mask=m)
  b.load_state_dict(a.state_dict())
  with torch.no_grad():
    rb = b(x, mask=m)
  assert all(torch.equal(p, q) for p, q in zip(ra, rb))


def test_input_checks():
  W, U = torch.zeros((4, 8), device="cuda"), torch.zeros((2, 8), device="cuda")
  with pytest.raises(ValueError, match="T = 0"):
    ops.lstm(torch.zeros((3, 0, 4), device="cuda"), W, U)
  out, h, c = ops.lstm(torch.zeros((0, 5, 4), device="cuda"), W, U, return_sequences=True)
  assert out.shape == (0, 5, 2) and h.shape == (0, 2) and c.shape == (0, 2)
  big = ops.LSTM_MAX_UNITS + 1
  with pytest.raises(ValueError, match=str(ops.LSTM_MAX_UNITS)):
    ops.lstm(torch.zeros((1, 1, 4), device="cuda"), torch.zeros((4, 4 * big), device="cuda"),
             torch.zeros((big, 4 * big), device="cuda"))
  with pytest.raises(ValueError, match=str(ops.LSTM_MAX_UNITS)):
    tfrs.layers.LSTM(big)
  with pytest.raises(ValueError, match="recurrent_kernel"):
    ops.lstm(torch.zeros((3, 5, 4), device="cuda"), W, torch.zeros((2, 6), device="cuda"))
  with pytest.raises(ValueError, match="bias"):
    ops.lstm(torch.zeros((3, 5, 4), device="cuda"), W, U, torch.zeros((2, 8), device="cuda"))
  with pytest.raises(ValueError, match="initial_state"):
    ops.lstm(torch.zeros((3, 5, 4), device="cuda"), W, U, initial_state=torch.zeros((3, 2), device="cuda"))
  with pytest.raises(ValueError, match="c_0"):
    ops.lstm(torch.zeros((3, 5, 4), device="cuda"), W, U,
             initial_state=(torch.zeros((3, 2), device="cuda"), torch.zeros((3, 3), device="cuda")))
  with pytest.raises(RuntimeError, match="CUDA"):
    ops.lstm(torch.zeros((3, 5, 4)), W, U)
  with pytest.raises(RuntimeError, match="CUDA"):
    ops.lstm(torch.zeros((3, 5, 4), device="cuda"), W, U,
             initial_state=(torch.zeros((3, 2), device="cuda"), torch.zeros((3, 2))))
  with pytest.raises(TypeError, match="lstm: the mask"):
    ops.lstm(torch.zeros((3, 5, 4), device="cuda"), W, U, mask=torch.ones((3, 5), device="cuda"))
  with pytest.raises(ValueError, match="lstm: the mask has shape"):
    ops.lstm(torch.zeros((3, 5, 4), device="cuda"), W, U, mask=torch.ones((3, 4), dtype=torch.bool, device="cuda"))
  with pytest.raises(NotImplementedError, match="return_sequences"):
    ops.lstm(torch.zeros((3, 5, 4), device="cuda"), W, U, mask=torch.ones((3, 5), dtype=torch.bool, device="cuda"),
             return_sequences=True)
  for kw in ({"activation": "relu"}, {"recurrent_activation": "hard_sigmoid"}, {"dropout": 0.5},
             {"recurrent_dropout": 0.5}, {"go_backwards": True}, {"stateful": True}, {"time_major": True}):
    with pytest.raises(NotImplementedError, match=next(iter(kw))):
      tfrs.layers.LSTM(4, **kw)


# ---- the sequential retrieval tutorial (docs/examples/sequential_retrieval.ipynb) with an LSTM(32) query tower -------
TUTORIAL_TOP10_FLOOR = 0.447  # half the held-out top-10 accuracy this seeded run reached on an H100 (0.8945)


def test_sequential_retrieval_tutorial_with_an_lstm_tower_trains_end_to_end(monkeypatch):
  def no_rnn(*a, **k):
    raise AssertionError("a torch / cuDNN RNN op ran")

  for mod in (torch, torch._VF):
    for name in ("gru", "gru_cell", "rnn_tanh", "rnn_relu", "lstm", "lstm_cell", "_cudnn_rnn"):
      if hasattr(mod, name):
        monkeypatch.setattr(mod, name, no_rnn)
  for cls in (torch.nn.GRU, torch.nn.GRUCell, torch.nn.RNN, torch.nn.LSTM, torch.nn.LSTMCell):
    monkeypatch.setattr(cls, "forward", no_rnn)

  ids, ctx, label = _histories()
  n_train = 49152
  torch.manual_seed(0)
  query_model = torch.nn.Sequential(tfrs.layers.StringLookup(vocabulary=ids, mask_token=None),
                                    Embedding(len(ids) + 1, 32), tfrs.layers.LSTM(32))
  candidate_model = torch.nn.Sequential(tfrs.layers.StringLookup(vocabulary=ids, mask_token=None),
                                        Embedding(len(ids) + 1, 32))
  movies = Dataset.from_tensor_slices(ids)
  task = tfrs.tasks.Retrieval(metrics=tfrs.metrics.FactorizedTopK(candidates=movies.batch(128).map(candidate_model)))
  model = _SequentialModel(query_model, candidate_model, task)
  model.compile(optimizer=tfrs.optimizers.Adagrad(learning_rate=0.1))
  train = Dataset.from_tensor_slices({"context_movie_id": ctx[:n_train], "label_movie_id": label[:n_train]}).batch(1024)
  test = Dataset.from_tensor_slices({"context_movie_id": ctx[n_train:], "label_movie_id": label[n_train:]}).batch(2560)

  before = model.evaluate(test)
  lstm = query_model[2]
  w0 = lstm.recurrent_kernel.detach().clone()
  hist = model.fit(train, epochs=3)
  after = model.evaluate(test)
  top10 = float(after["factorized_top_k/top_10_categorical_accuracy"])
  print(f"sequential tutorial (LSTM): loss {float(before['loss']):.4f} -> {float(after['loss']):.4f}, "
        f"held-out top-10 accuracy {float(before['factorized_top_k/top_10_categorical_accuracy']):.4f} -> {top10:.4f}")
  assert all(np.isfinite(float(h["loss"])) for h in hist)
  assert float(after["loss"]) < float(before["loss"])
  assert top10 >= TUTORIAL_TOP10_FLOOR
  # the LSTM's weights are ordinary dense parameters: Adagrad moved them
  assert not torch.equal(w0, lstm.recurrent_kernel.detach())
