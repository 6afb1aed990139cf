"""K21 / K22 on the H100: `ops.attention` / `layers.MultiHeadAttention` and `ops.layer_norm` / `layers.LayerNormalization`
against the float64 oracle (tests/attention_oracle.py) over lengths, every staged-tile edge, cross attention,
heads, head dims, every mask source and mask dtype, fully masked rows and the returned scores; row widths and flags of
the normalization; bitwise invariances; launch counts; input errors; and the sequential retrieval tutorial with a
one-block SASRec query tower trained end to end."""
import math

import numpy as np
import pytest
import torch

import attention_oracle as ao
import recommenders_b200 as tfrs
from recommenders_b200 import ops
from recommenders_b200.data import Dataset
from recommenders_b200.layers.attention import keras_fans
from recommenders_b200.layers.blocks import Dense
from recommenders_b200.layers.embedding import Embedding
from test_gpu_gru import _SequentialModel, _histories

pytestmark = pytest.mark.gpu

MASK_DTYPES = {"bool": torch.bool, "int32": torch.int32, "int64": torch.int64}


def _plan(L, width):
  """Rows staged per sequence (csrc/attention.cu mha_plan) when a CTA's 32 rows have length L."""
  nseq = min((31 + L - 1) // L + 1, 32)
  return max(1, min(64, 65536 // (nseq * width * 4)))


BASE = [1, 2, 31, 32, 33, 63, 64, 65, 127, 128, 129, 200, 513]


def _lengths(dk, dv):
  tiles = {_plan(L, dk + dv) for L in BASE} | {_plan(L, dk + dv + 3) for L in BASE}
  return sorted(set(BASE) | {t + e for t in tiles for e in (-1, 0, 1) if t + e >= 1})


def _cu(a, grad=False, dtype=None):
  if a is None:
    return None
  t = torch.from_numpy(np.ascontiguousarray(a)).cuda()
  return (t.to(dtype) if dtype is not None else t).requires_grad_(grad)


def _check(name, got, exp, bar=1e-5, scale=None):
  got = got.detach().double().cpu().numpy() if isinstance(got, torch.Tensor) else got
  assert got.shape == exp.shape, (name, got.shape, exp.shape)
  if scale is None:
    scale = np.abs(exp).max() if exp.size else 0.0
  err = np.abs(got - exp).max() if exp.size else 0.0
  assert err <= bar * scale, f"{name}: max |error| {err:.3g} > {bar:g} * max |value| {scale:.3g}"


def _glorot(rng, shape):
  fi, fo = keras_fans(shape)
  return rng.uniform(-1, 1, size=shape).astype(np.float32) * np.float32(math.sqrt(6 / (fi + fo)))


def _masks(kinds, B, T, S, rng, dtype="bool"):
  """numpy masks by source: "query", "value", "key", "attention" (random), "causal"; "qfull" masks whole query rows."""
  m = {}
  for k in kinds:
    if k == "query":
      m["query_mask"] = rng.rand(B, T) < 0.7
    elif k == "qfull":
      q = np.ones((B, T), bool)
      q[:, ::3] = False
      m["query_mask"] = q
    elif k == "value":
      m["value_mask"] = rng.rand(B, S) < 0.6
    elif k == "key":
      m["key_mask"] = rng.rand(B, S) < 0.7
    elif k == "attention":
      m["attention_mask"] = rng.rand(B, T, S) < 0.5
  return m


def _run(B, T, S, H, dk, dv, masks=(), dtype="bool", causal=False, cross_key=True, bias=True, scores=False, seed=0,
         Dq=24, Dv=20, Dk=12, Dout=None):
  rng = np.random.RandomState(seed)
  Dout = Dout or Dq
  query = rng.normal(size=(B, T, Dq)).astype(np.float32)
  value = rng.normal(size=(B, S, Dv)).astype(np.float32)
  key = rng.normal(size=(B, S, Dk)).astype(np.float32) if cross_key else None
  W = [_glorot(rng, s) for s in ((Dq, H, dk), (Dk if cross_key else Dv, H, dk), (Dv, H, dv), (H, dv, Dout))]
  b = ([(rng.normal(size=s) * 0.1).astype(np.float32) for s in ((H, dk), (H, dk), (H, dv), (Dout,))] if bias
       else [None] * 4)
  m = _masks(masks, B, T, S, rng)
  g = rng.normal(size=(B, T, Dout)).astype(np.float32)
  ts = [_cu(a, True) for a in (query, value, key, *W, *b)]
  mt = {k: _cu(v, dtype=MASK_DTYPES[dtype]) for k, v in m.items()}
  out, P = ops.attention(*ts[:3], *ts[3:7], *ts[7:], causal=causal, return_scores=scores, **mt)
  (out * _cu(g)).sum().backward()

  keep = ao.combined_mask(B, T, S, causal=causal, **m)
  eout, eP, cache = ao.mha_forward(query, value, key, *W, *b, keep=keep)
  r = ao.mha_backward(cache, g, key_is_value=key is None)
  _check("out", out, eout)
  if scores:
    assert not P.requires_grad
    _check("scores", P, eP)
  _check("dquery", ts[0].grad, r["dquery"])
  _check("dvalue", ts[1].grad, r["dvalue"])
  if key is not None:
    _check("dkey", ts[2].grad, r["dkey"])
  for i, n in enumerate("qkvo"):
    _check("dW" + n, ts[3 + i].grad, r["dW" + n])
  if bias:
    for i, n in enumerate("qvo"):
      _check("db" + n, ts[7 + "qkvo".index(n)].grad, r["db" + n])
    # dbk is exactly zero: the fp32 result is the cancellation of sum_{b,s} dK, so its bar is 1e-5 of the summed
    # magnitudes sum_{b,s} |dK| (each term within the dK bar), not of the zero it cancels to
    _check("dbk", ts[8].grad, r["dbk"], scale=r["dbk_terms"].max())
  return keep


def test_the_tile_edges_are_in_the_length_grid():
  L = _lengths(16, 16)
  assert {63, 64, 65} <= set(L) and _plan(10, 32) == 64 and _plan(1, 32) == 16
  assert {15, 16, 17} <= set(L)


def _tile_edge_pairs(dk, dv):
  """(T, S) pairs whose walked side sits at a planned tile - 1, tile, tile + 1: the forward and dQ kernels walk S in
  tiles planned from T (width dk + dv), the dK / dV kernel walks T in tiles planned from S (width dk + dv + 3)."""
  pairs = set()
  for L in BASE + [10]:                             # and the tutorial's T = 10
    pairs |= {(L, _plan(L, dk + dv) + e) for e in (-1, 0, 1)}
    pairs |= {(_plan(L, dk + dv + 3) + e, L) for e in (-1, 0, 1)}
  return sorted((t, s) for t, s in pairs if t >= 1 and s >= 1)


def test_the_edge_pairs_cross_the_short_sequence_tiles():
  pairs = set(_tile_edge_pairs(16, 16))
  assert {(1, 15), (1, 16), (1, 17), (2, 29), (2, 30), (2, 31), (10, 65)} <= pairs        # forward / dQ walks over S
  assert {(13, 1), (14, 1), (15, 1), (26, 2), (27, 2), (28, 2), (65, 10)} <= pairs        # dK / dV walks over T


@pytest.mark.parametrize("T,S", _tile_edge_pairs(16, 16))
def test_every_staged_tile_edge_matches_the_oracle(T, S):
  _run(2, T, S, 2, 16, 16, masks=("value",), causal=True, seed=T * 1000 + S)


# with T = S the tile is planned from the length itself: these cover the lengths, the pairs above the tile edges
@pytest.mark.parametrize("T", _lengths(16, 16))
def test_self_attention_lengths_match_the_oracle(T):
  _run(2, T, T, 2, 16, 16, causal=True, cross_key=False, seed=T)


@pytest.mark.parametrize("T,S", [(1, 513), (513, 1), (10, 200), (200, 10), (33, 65), (65, 33), (17, 129), (129, 2)])
def test_cross_attention_lengths_match_the_oracle(T, S):
  _run(3, T, S, 2, 16, 16, masks=("value",), seed=T * 1000 + S)


@pytest.mark.parametrize("dk,dv,H", [(1, 128, 1), (8, 100, 2), (16, 64, 8), (31, 32, 1), (32, 31, 2), (64, 16, 8),
                                     (100, 8, 1), (128, 1, 2), (128, 128, 8)])
def test_head_dims_and_heads_match_the_oracle(dk, dv, H):
  _run(2, 33, 65, H, dk, dv, masks=("key",), seed=dk * 1000 + dv)
  _run(2, 65, 17, H, dk, dv, causal=True, cross_key=False, seed=dk * 1000 + dv + 1)


@pytest.mark.parametrize("masks,causal", [((), False), (("query",), False), (("value",), False), (("key",), False),
                                          (("attention",), False), ((), True),
                                          (("query", "value", "key", "attention"), True), (("qfull", "value"), True)])
@pytest.mark.parametrize("dtype", ["bool", "int32", "int64"])
def test_every_mask_source_and_dtype_matches_the_oracle(masks, causal, dtype):
  keep = _run(3, 20, 24, 2, 8, 12, masks=masks, causal=causal, dtype=dtype, scores=True, seed=len(masks) * 7 + causal)
  if "qfull" in masks:
    assert not keep[:, ::3].any()                   # fully masked rows: uniform attention, checked against the oracle


def test_fully_masked_rows_and_the_returned_scores():
  B, T, S = 2, 6, 9
  rng = np.random.RandomState(3)
  vm = np.ones((B, S), bool)
  vm[1] = False                                     # every row of batch 1 fully masked
  Q, K, V = (_cu(rng.normal(size=(B, n, 2 * 4)).astype(np.float32)) for n in (T, S, S))
  with torch.no_grad():
    O, P = ops.attention_core(Q, K, V, 2, value_mask=_cu(vm), return_scores=True)
  # l = S exactly; P = e^0 / l through __fdividef (2 ulp)
  assert torch.allclose(P[1], torch.full((2, T, S), 1.0 / S, device="cuda"), rtol=2.5e-7, atol=0)
  _check("uniform O", O[1], V[1].double().cpu().numpy().mean(0)[None].repeat(T, 0))


def test_return_scores_and_no_grad_outputs_are_bitwise_equal_to_grad_mode():
  rng = np.random.RandomState(5)
  B, T, S, H, d = 4, 37, 41, 2, 16
  Q, K, V = (rng.normal(size=(B, n, H * d)).astype(np.float32) for n in (T, S, S))
  am = _cu(rng.rand(B, T, S) < 0.5)
  with torch.no_grad():
    O0, P0 = ops.attention_core(_cu(Q), _cu(K), _cu(V), H, attention_mask=am, causal=True, return_scores=True)
  O1, P1 = ops.attention_core(_cu(Q, True), _cu(K, True), _cu(V, True), H, attention_mask=am, causal=True,
                              return_scores=True)
  O2, _ = ops.attention_core(_cu(Q, True), _cu(K, True), _cu(V, True), H, attention_mask=am, causal=True)
  assert O1.requires_grad and not P1.requires_grad
  assert torch.equal(O0, O1.detach()) and torch.equal(P0, P1) and torch.equal(O0, O2.detach())
  x = rng.normal(size=(300, 129)).astype(np.float32)
  with torch.no_grad():
    y0 = ops.layer_norm(_cu(x), _cu(np.ones(129, np.float32)), _cu(np.zeros(129, np.float32)))
  y1 = ops.layer_norm(_cu(x, True), _cu(np.ones(129, np.float32), True), _cu(np.zeros(129, np.float32), True))
  assert torch.equal(y0, y1.detach())


def test_two_identical_training_steps_are_bitwise_equal():
  rng = np.random.RandomState(9)
  B, T, D = 64, 50, 32

  def step():
    torch.manual_seed(0)
    mha, ln = tfrs.layers.MultiHeadAttention(4, 8), tfrs.layers.LayerNormalization()
    x = _cu(rng.normal(size=(B, T, D)).astype(np.float32), True)
    y = ln(x + mha(x, x, use_causal_mask=True))
    (y * y).sum().backward()
    return [y.detach(), x.grad] + [p.grad for p in (*mha.parameters(), *ln.parameters())]

  state = rng.get_state()
  a = step()
  rng.set_state(state)
  for u, v in zip(a, step()):
    assert torch.equal(u, v)


@pytest.mark.parametrize("T", [1, 513])
def test_launch_counts(T):
  rng = np.random.RandomState(T)
  Q, K, V = (_cu(rng.normal(size=(2, T, 32)).astype(np.float32), True) for _ in range(3))
  n = ops.launch_count()
  O, _ = ops.attention_core(Q, K, V, 2, causal=True)
  assert ops.launch_count() - n == 1
  n = ops.launch_count()
  O.sum().backward()
  assert ops.launch_count() - n <= 3
  with torch.no_grad():
    n = ops.launch_count()
    ops.attention_core(Q, K, V, 2, return_scores=True)
    assert ops.launch_count() - n == 1
  x = _cu(rng.normal(size=(T, 64)).astype(np.float32), True)
  g, b = _cu(np.ones(64, np.float32), True), _cu(np.zeros(64, np.float32), True)
  n = ops.launch_count()
  y = ops.layer_norm(x, g, b)
  assert ops.launch_count() - n == 1
  n = ops.launch_count()
  y.sum().backward()
  assert ops.launch_count() - n == 2


# ---- LayerNormalization -------------------------------------------------------------------------------------------
WIDTHS = [1, 2, 31, 32, 33, 127, 128, 129, 1000, 1024, 4096]


def _ln_case(N, d, center=True, scale=True, offset=0.0, seed=0, lead=None):
  rng = np.random.RandomState(seed)
  shape = lead + (d,) if lead else (N, d)
  x = (rng.normal(size=shape) + offset).astype(np.float32)
  gamma = rng.normal(size=d).astype(np.float32) if scale else None
  beta = rng.normal(size=d).astype(np.float32) if center else None
  g = rng.normal(size=shape).astype(np.float32)
  xt, gt, bt = _cu(x, True), _cu(gamma, True), _cu(beta, True)
  y = ops.layer_norm(xt, gt, bt, 1e-3)
  (y * _cu(g)).sum().backward()
  ey, _, _ = ao.layer_norm_forward(x, gamma, beta)
  dx, dg, db = ao.layer_norm_backward(x, gamma, g)
  _check("y", y, ey)
  _check("dx", xt.grad, dx)
  if scale:
    _check("dgamma", gt.grad, dg)
  if center:
    _check("dbeta", bt.grad, db)


@pytest.mark.parametrize("d", WIDTHS)
@pytest.mark.parametrize("N", [0, 1, 37, 3000])
def test_layer_norm_widths_and_rows_match_the_oracle(d, N):
  _ln_case(N, d, seed=d * 7 + N)


@pytest.mark.parametrize("center,scale", [(False, True), (True, False), (False, False)])
def test_layer_norm_without_center_or_scale(center, scale):
  _ln_case(257, 65, center, scale, seed=4)
  _ln_case(0, 65, center, scale, seed=4, lead=(0, 3))


@pytest.mark.parametrize("d", [32, 1024, 4096])
def test_layer_norm_rows_with_mean_1e4_and_std_1(d):
  _ln_case(200, d, offset=1e4, seed=d)


def test_layer_norm_on_a_3d_input_and_the_layer():
  _ln_case(0, 48, seed=2, lead=(5, 7))
  rng = np.random.RandomState(1)
  ids = rng.randint(0, 20, size=(4, 6))
  e = Embedding(20, 8, mask_zero=True)(torch.from_numpy(ids).cuda())
  ln = tfrs.layers.LayerNormalization(epsilon=1e-5)
  y = ln(e)
  assert torch.equal(ops.attached_mask(y), ops.attached_mask(e))
  ey, _, _ = ao.layer_norm_forward(e.detach().cpu().numpy(), ln.gamma.detach().cpu().numpy(),
                                   ln.beta.detach().cpu().numpy(), 1e-5)
  _check("layer y", y, ey)


# ---- the layer, masks carried by Embedding outputs, and input errors ----------------------------------------------
def test_the_layer_with_attached_masks_and_config():
  torch.manual_seed(0)
  B, T, S, n, d = 8, 7, 9, 30, 16
  rng = np.random.RandomState(6)
  qi, vi = rng.randint(0, n, size=(B, T)), rng.randint(0, n, size=(B, S))
  qi[rng.rand(B, T) < 0.3] = 0
  vi[rng.rand(B, S) < 0.3] = 0
  emb = Embedding(n, d, mask_zero=True)
  q, v = emb(torch.from_numpy(qi).cuda()), emb(torch.from_numpy(vi).cuda())
  layer = tfrs.layers.MultiHeadAttention(2, 8, value_dim=6, output_shape=10)
  out, P = layer(q, v, return_attention_scores=True)
  assert out.shape == (B, T, 10) and P.shape == (B, 2, T, S)
  assert ops.attached_mask(out) is not None and torch.equal(ops.attached_mask(out), ops.attached_mask(q))
  W = [w.detach().cpu().numpy() for w in (layer.query.kernel, layer.key.kernel, layer.value.kernel,
                                           layer.attention_output.kernel, layer.query.bias, layer.key.bias,
                                           layer.value.bias, layer.attention_output.bias)]
  keep = ao.combined_mask(B, T, S, query_mask=qi, value_mask=vi)
  eout, eP, _ = ao.mha_forward(q.detach().cpu().numpy(), v.detach().cpu().numpy(), None, *W, keep=keep)
  _check("layer out", out, eout)
  _check("layer scores", P, eP)
  # the Keras 3 keywords stand in for a mask a residual add dropped
  out2 = layer(q + 0, v + 0, query_mask=torch.from_numpy(qi).cuda(), value_mask=torch.from_numpy(vi != 0).cuda())
  assert torch.equal(out2, out)
  again = tfrs.layers.MultiHeadAttention.from_config(layer.get_config())
  assert again.get_config() == layer.get_config()


def test_input_checks():
  x = torch.zeros((2, 3, 8), device="cuda")
  with pytest.raises(ValueError, match="128"):
    ops.attention_core(torch.zeros((2, 3, 129), device="cuda"), torch.zeros((2, 3, 129), device="cuda"),
                       torch.zeros((2, 3, 8), device="cuda"), 1)
  with pytest.raises(ValueError, match="128"):
    tfrs.layers.MultiHeadAttention(2, 129)
  with pytest.raises(ValueError, match="heads"):
    ops.attention_core(x, x, x, 3)
  with pytest.raises(ValueError, match="query_mask"):
    ops.attention_core(x, x, x, 2, query_mask=torch.ones((2, 4), dtype=torch.bool, device="cuda"))
  with pytest.raises(ValueError, match="attention_mask"):
    ops.attention_core(x, x, x, 2, attention_mask=torch.ones((2, 3), dtype=torch.bool, device="cuda"))
  with pytest.raises(TypeError, match="value_mask"):
    ops.attention_core(x, x, x, 2, value_mask=torch.ones((2, 3), device="cuda"))
  with pytest.raises(RuntimeError, match="CUDA"):
    ops.attention_core(x, x, x, 2, key_mask=torch.ones((2, 3), dtype=torch.bool))
  with pytest.raises(ValueError, match="empty"):
    ops.attention_core(torch.zeros((2, 0, 8), device="cuda"), x, x, 2)
  with pytest.raises(ValueError, match="do not fit"):
    ops.attention_core(x, torch.zeros((2, 4, 6), device="cuda"), torch.zeros((2, 4, 8), device="cuda"), 2)
  layer = tfrs.layers.MultiHeadAttention(2, 4)
  with pytest.raises(NotImplementedError, match="rank"):
    layer(torch.zeros((2, 3, 4, 8), device="cuda"), torch.zeros((2, 3, 4, 8), device="cuda"))
  layer(x, x)
  with pytest.raises(ValueError, match="kernel"):
    layer(torch.zeros((2, 3, 5), device="cuda"), x)
  O, P = ops.attention_core(torch.zeros((0, 3, 8), device="cuda"), torch.zeros((0, 4, 8), device="cuda"),
                            torch.zeros((0, 4, 8), device="cuda"), 2, return_scores=True)
  assert O.shape == (0, 3, 8) and P.shape == (0, 2, 3, 4)
  with pytest.raises(ValueError, match="gamma"):
    ops.layer_norm(x, torch.ones(7, device="cuda"))
  with pytest.raises(RuntimeError, match="CUDA"):
    ops.layer_norm(x, torch.ones(8))


# ---- the sequential retrieval tutorial with a one-block SASRec query tower ----------------------------------------
TUTORIAL_TOP10_FLOOR = 0.451  # half the held-out top-10 accuracy this seeded run reached on an H100 (0.9023)


class _SASRec(torch.nn.Module):
  """StringLookup -> item Embedding(301, 32) + position Embedding(10, 32) -> causal MultiHeadAttention(2, 16), residual,
  LayerNormalization -> Dense(64, relu) -> Dense(32), residual, LayerNormalization -> the last position."""

  def __init__(self, ids, T=10, d=32):
    super().__init__()
    self.lookup = tfrs.layers.StringLookup(vocabulary=ids, mask_token=None)
    self.item, self.position = Embedding(len(ids) + 1, d), Embedding(T, d)
    self.attention = tfrs.layers.MultiHeadAttention(2, 16)
    self.norm1, self.norm2 = tfrs.layers.LayerNormalization(), tfrs.layers.LayerNormalization()
    self.ff1, self.ff2 = Dense(64, activation="relu"), Dense(d)

  def forward(self, history):
    ids = self.lookup(history)
    B, T = ids.shape
    x = self.item(ids) + self.position(torch.arange(T, device=ids.device).expand(B, T))
    x = self.norm1(x + self.attention(x, x, use_causal_mask=True))
    x = self.norm2(x + self.ff2(self.ff1(x)))
    return x[:, -1]


def test_sequential_retrieval_tutorial_with_a_sasrec_tower_trains_end_to_end(monkeypatch):
  def banned(*a, **k):
    raise AssertionError("a torch attention / softmax / layer_norm / matmul op ran")

  F = torch.nn.functional
  for mod, names in ((F, ("scaled_dot_product_attention", "softmax", "layer_norm", "multi_head_attention_forward")),
                     (torch, ("softmax", "layer_norm", "bmm", "baddbmm", "matmul", "einsum")),
                     (torch.Tensor, ("softmax", "matmul", "__matmul__", "bmm", "baddbmm"))):
    for name in names:
      if hasattr(mod, name):
        monkeypatch.setattr(mod, name, banned)
  monkeypatch.setattr(torch.nn.MultiheadAttention, "forward", banned)

  ids, ctx, label = _histories()
  n_train = 49152
  torch.manual_seed(0)
  query_model = _SASRec(ids)
  candidate_model = torch.nn.Sequential(tfrs.layers.StringLookup(vocabulary=ids, mask_token=None),
                                        Embedding(len(ids) + 1, 32))
  movies = Dataset.from_tensor_slices(ids)
  task = tfrs.tasks.Retrieval(metrics=tfrs.metrics.FactorizedTopK(candidates=movies.batch(128).map(candidate_model)))
  model = _SequentialModel(query_model, candidate_model, task)
  model.compile(optimizer=tfrs.optimizers.Adagrad(learning_rate=0.1))
  train = Dataset.from_tensor_slices({"context_movie_id": ctx[:n_train], "label_movie_id": label[:n_train]}).batch(1024)
  test = Dataset.from_tensor_slices({"context_movie_id": ctx[n_train:], "label_movie_id": label[n_train:]}).batch(2560)

  before = model.evaluate(test)
  w0 = query_model.attention.query.kernel.detach().clone()
  hist = model.fit(train, epochs=3)
  after = model.evaluate(test)
  top10 = float(after["factorized_top_k/top_10_categorical_accuracy"])
  print(f"sequential tutorial (SASRec): loss {float(before['loss']):.4f} -> {float(after['loss']):.4f}, "
        f"held-out top-10 accuracy {float(before['factorized_top_k/top_10_categorical_accuracy']):.4f} -> {top10:.4f}")
  assert all(np.isfinite(float(h["loss"])) for h in hist)
  assert float(after["loss"]) < float(before["loss"])
  assert top10 >= TUTORIAL_TOP10_FLOOR
  # the attention weights are ordinary dense parameters: Adagrad moved them
  assert not torch.equal(w0, query_model.attention.query.kernel.detach())
