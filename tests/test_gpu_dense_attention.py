"""K21's dot scores and K25's tanh scores on the H100: `ops.dense_attention` / `layers.Attention` /
`layers.AdditiveAttention` against the float64 oracle (tests/dense_attention_oracle.py) over the three score modes with
and without scale, head dims, lengths at every staged-tile edge, the 32-row CTA edge, every mask source and dtype, fully
masked rows and dropout rates; the dropout mask bit for bit; launch counts and bitwise repeatability; and a DIN-style
ranking model trained end to end."""
import math

import numpy as np
import pytest
import torch

import dense_attention_oracle as dao
import recommenders_b200 as tfrs
import regularization_oracle as ro
from recommenders_b200 import ops
from recommenders_b200.data import Dataset
from recommenders_b200.layers import AdditiveAttention, Attention
from recommenders_b200.layers.embedding import Embedding
from test_gpu_gru import _histories
from test_gpu_regularization import _ban

pytestmark = pytest.mark.gpu

MASK_DTYPES = {"bool": torch.bool, "int32": torch.int32, "int64": torch.int64}


def _plan(L, width):
  """Rows staged per sequence (csrc/attention.cuh mha_plan) when a CTA's 32 rows have length L."""
  nseq = min((31 + L - 1) // L + 1, 32)
  return max(1, min(64, 65536 // (nseq * width * 4)))


def _edges(dim, dv):
  """1, 513 and every staged-tile size +-1 the forward / dQ (width dim + dv) and dK / dV (dim + dv + 3) plans take."""
  base = [1, 2, 31, 32, 33, 63, 64, 65, 127, 128, 129, 200, 513]
  tiles = {_plan(L, dim + dv) for L in base} | {_plan(L, dim + dv + 3) for L in base}
  return sorted({1, 513} | {t + e for t in tiles for e in (-1, 0, 1) if t + e >= 1})


def _check(name, got, exp, bar=1e-5, scale=None):
  got = got.detach().double().cpu().numpy() if isinstance(got, torch.Tensor) else np.asarray(got, np.float64)
  exp = np.asarray(exp, np.float64)
  assert got.size == exp.size, (name, got.shape, exp.shape)
  got = got.reshape(exp.shape)
  if scale is None:
    scale = np.abs(exp).max() if exp.size else 0.0
  err = np.abs(got - exp).max() if exp.size else 0.0
  assert err <= bar * scale, f"{name}: max |error| {err:.3g} > {bar:g} * max |value| {scale:.3g}"


def _weights(rng, mode, use_scale, dim):
  scale = cw = None
  if use_scale:
    if mode == "additive":
      lim = math.sqrt(3.0 / dim)
      scale = rng.uniform(-lim, lim, size=(dim,)).astype(np.float32)
    else:
      scale = np.array(rng.uniform(0.5, 1.5), np.float32)
  if mode == "concat":
    cw = np.array(rng.uniform(0.5, 1.5), np.float32)
  return scale, cw


def _case(mode, use_scale, B, Tq, Tv, dim, dv, qm=None, vm=None, causal=False, rate=0.0, seed=5, call=0,
          key_is_value=False, mask_dtype="bool", seed_data=0):
  """Run ops.dense_attention forward and backward and hold every output and gradient to the oracle."""
  rng = np.random.RandomState(seed_data)
  u = dim ** -0.25                                 # q . k of order 1, as with embeddings of Keras's initial scale
  q = (rng.normal(size=(B, Tq, dim)) * u).astype(np.float32)
  v = (rng.normal(size=(B, Tv, dv)) * (u if key_is_value else 1.0)).astype(np.float32)
  k = v if key_is_value else (rng.normal(size=(B, Tv, dim)) * u).astype(np.float32)
  scale, cw = _weights(rng, mode, use_scale, dim)
  g = rng.normal(size=(B, Tq, dv)).astype(np.float32)
  cu = lambda a: None if a is None else torch.from_numpy(np.ascontiguousarray(a)).cuda().requires_grad_(True)
  tq, tv = cu(q), cu(v)
  tk = tv if key_is_value else cu(k)
  ts, tw = cu(scale), cu(cw)
  dt = MASK_DTYPES[mask_dtype]
  mk = lambda m: None if m is None else torch.from_numpy(np.asarray(m)).cuda().to(dt)
  out, w = ops.dense_attention(tq, tk, tv, mode, ts, tw, query_mask=mk(qm), value_mask=mk(vm), causal=causal,
                               rate=rate, seed=seed, call=call, return_scores=True)
  out.backward(torch.from_numpy(g).cuda())
  keep = ro.dropout_keep((B, Tq, Tv), rate, seed, call) if rate else None
  eo, ew, cache = dao.forward(q, k, v, mode, scale, cw, qm, vm, causal, keep, rate)
  dq, dk, dv_, dscale, dwc = dao.backward(cache, g)
  _check("out", out, eo)
  _check("weights", w, ew)
  _check("dq", tq.grad, dq)
  if key_is_value:
    _check("dv (key = value)", tv.grad, dk + dv_)
  else:
    _check("dk", tk.grad, dk)
    _check("dv", tv.grad, dv_)
  # A scalar weight gradient sums B * Tq rows whose contributions cancel (each row's ds sums to 0), so it is held to
  # 1e-5 of the sum of the rows' magnitudes where that is larger than its own
  rows_scale, rows_wc = dao.weight_grad_rows(cache, g)
  l1 = lambda r, e: max(np.abs(e).max(), np.abs(r).sum()) if r is not None else None
  if use_scale:
    _check("dscale", ts.grad, dscale, scale=l1(rows_scale, dscale))
  if mode == "concat":
    _check("dconcat_weight", tw.grad, dwc, scale=l1(rows_wc, dwc))
  return w


DIMS = [1, 7, 8, 31, 32, 33, 64, 100, 128]


@pytest.mark.parametrize("mode", dao.MODES)
@pytest.mark.parametrize("use_scale", [False, True])
@pytest.mark.parametrize("i", range(len(DIMS)))
def test_every_mode_and_dim(mode, use_scale, i):
  dim, dv = DIMS[i], DIMS[(i + 4) % len(DIMS)]
  _case(mode, use_scale, 3, 5, 9, dim, dv, seed_data=i)


LENGTHS = _edges(32, 24)


@pytest.mark.parametrize("mode", dao.MODES)
@pytest.mark.parametrize("L", LENGTHS)
def test_lengths_at_every_tile_edge(mode, L):
  rng = np.random.RandomState(L)
  _case(mode, True, 2, 1, L, 32, 24, vm=rng.rand(2, L) < 0.8, seed_data=L)            # target attention
  _case(mode, True, 2, L, L, 32, 24, qm=rng.rand(2, L) < 0.8, causal=True, seed_data=L + 1)   # self attention
  _case(mode, False, 2, L, 3, 32, 24, seed_data=L + 2)


@pytest.mark.parametrize("B,Tq", [(31, 1), (32, 1), (33, 1), (5, 7), (1, 31), (1, 33), (3, 11), (65, 1)])
def test_query_rows_across_the_cta_edge(B, Tq):
  for mode in dao.MODES:
    rng = np.random.RandomState(B * Tq)
    _case(mode, True, B, Tq, 6, 16, 8, qm=rng.rand(B, Tq) < 0.7, vm=rng.rand(B, 6) < 0.7, rate=0.3, call=B,
          seed_data=B + Tq)


@pytest.mark.parametrize("mode", dao.MODES)
def test_weight_gradients_at_training_size(mode):
  """20480 query rows (a BST-sized batch), masked and dropped out: the weight gradients' folds over every row."""
  rng = np.random.RandomState(21)
  B, Tq, Tv = 2048, 10, 12
  _case(mode, True, B, Tq, Tv, 32, 16, vm=rng.rand(B, Tv) < 0.8, rate=0.1, call=4, seed_data=21)


@pytest.mark.parametrize("mask_dtype", list(MASK_DTYPES))
@pytest.mark.parametrize("which", ["query", "value", "both", "full_rows"])
def test_masks_of_every_source_and_dtype(mask_dtype, which):
  B, Tq, Tv = 4, 6, 7
  rng = np.random.RandomState(2)
  qm = rng.rand(B, Tq) < 0.6 if which in ("query", "both", "full_rows") else None
  vm = rng.rand(B, Tv) < 0.6 if which in ("value", "both", "full_rows") else None
  if which == "full_rows":
    qm[1] = False                                  # a fully masked query row: a zero output row, no gradient
    vm[2] = False                                  # a fully masked value row: uniform weights
  for mode in dao.MODES:
    for causal in (False, True):
      _case(mode, True, B, Tq, Tv, 12, 12 if causal else 5, qm=qm, vm=vm, causal=causal, mask_dtype=mask_dtype,
            key_is_value=causal)


@pytest.mark.parametrize("rate", [0.0, 2.0 ** -24, 0.1, 0.5, 0.999])
@pytest.mark.parametrize("mode", dao.MODES)
def test_dropout_rates(rate, mode):
  rng = np.random.RandomState(9)
  w = _case(mode, True, 6, 9, 70, 20, 12, qm=rng.rand(6, 9) < 0.8, vm=rng.rand(6, 70) < 0.8, rate=rate, seed=77,
            call=3)
  if rate:
    keep = ro.dropout_keep((6, 9, 70), rate, 77, 3)
    wn = w.cpu().numpy()
    assert np.all(wn[~keep] == 0) and not np.signbit(wn[~keep]).any(), "a dropped weight is not +0"


def _layer_pair(mode, **kw):
  return Attention(score_mode=mode, **kw) if mode != "additive" else AdditiveAttention(**kw)


@pytest.mark.parametrize("mode", dao.MODES)
def test_layer_training_and_inference(mode):
  """Dropout only in training; at inference and at rate 0 the weights are the plain softmax, no RNG, one launch."""
  rng = np.random.RandomState(4)
  q = torch.from_numpy(rng.normal(size=(8, 3, 16)).astype(np.float32)).cuda()
  v = torch.from_numpy(rng.normal(size=(8, 20, 16)).astype(np.float32)).cuda()
  layer = _layer_pair(mode, use_scale=True, dropout=0.4, seed=123)
  plain = _layer_pair(mode, use_scale=True)
  plain(([q, v]))
  with torch.no_grad():
    layer([q, v])
    plain.load_state_dict(layer.state_dict())
    state = torch.cuda.get_rng_state()
    n0 = ops.launch_count()
    o_inf, w_inf = layer([q, v], return_attention_scores=True)
    assert ops.launch_count() - n0 == 1
    o_plain, w_plain = plain([q, v], return_attention_scores=True, training=True)
    assert torch.equal(o_inf, o_plain) and torch.equal(w_inf, w_plain)
    assert layer._calls == 0 and plain._calls == 0
    n0 = ops.launch_count()
    _, w1 = layer([q, v], training=True, return_attention_scores=True)
    assert ops.launch_count() - n0 == 1
    _, w2 = layer([q, v], training=True, return_attention_scores=True)
    assert layer._calls == 2 and not torch.equal(w1, w2), "successive training calls drew the same mask"
    assert torch.equal(state, torch.cuda.get_rng_state())
    keep = ro.dropout_keep((8, 3, 20), 0.4, 123, 1)
    assert np.array_equal(w2.cpu().numpy() != 0, keep & (w_inf.cpu().numpy() != 0))
    again = _layer_pair(mode, use_scale=True, dropout=0.4, seed=123)
    again([q, v])
    again.load_state_dict(layer.state_dict())
    _, a1 = again([q, v], training=True, return_attention_scores=True)
    assert torch.equal(a1, w1), "a seeded layer did not repeat its masks"


@pytest.mark.parametrize("mode", dao.MODES)
def test_two_identical_training_steps_are_bitwise_equal(mode):
  rng = np.random.RandomState(8)
  data = [rng.normal(size=s).astype(np.float32) for s in ((64, 5, 32), (64, 50, 32), (64, 5, 32))]

  def step():
    q, v, g = (torch.from_numpy(a).cuda().requires_grad_(True) for a in data)
    layer = _layer_pair(mode, use_scale=True, dropout=0.1, seed=1)
    layer.build(32, q.device)
    if layer.scale is not None and mode == "additive":
      with torch.no_grad():
        layer.scale.copy_(torch.linspace(-0.3, 0.3, 32, device=q.device))
    n0 = ops.launch_count()
    out = layer([q, v], training=True)
    n1 = ops.launch_count()
    out.backward(g)
    n2 = ops.launch_count()
    assert n1 - n0 == 1
    assert n2 - n1 == 3 + 1 + (mode == "concat"), "backward: delta, dK / dV, dQ and one fold per weight gradient"
    grads = [q.grad, v.grad] + [p.grad for p in layer.parameters()]
    return [t.detach().cpu().numpy().view(np.uint32) for t in [out] + grads]

  a, b = step(), step()
  assert all(np.array_equal(x, y) for x, y in zip(a, b))


def test_attached_masks_and_output_mask():
  rng = np.random.RandomState(6)
  emb = Embedding(50, 16, mask_zero=True)
  ids_q = torch.from_numpy(rng.randint(0, 50, size=(4, 3))).cuda()
  ids_v = torch.from_numpy(rng.randint(0, 50, size=(4, 9))).cuda()
  ids_q[0] = 0
  ids_v[1] = 0
  for mode in dao.MODES:
    layer = _layer_pair(mode, use_scale=True)
    with torch.no_grad():
      xq, xv = emb(ids_q), emb(ids_v)
      out, w = layer([xq, xv], return_attention_scores=True)
    assert torch.equal(ops.attached_mask(out) != 0, ids_q != 0)
    p = {n: t.detach().cpu().numpy() for n, t in layer.named_parameters()}
    eo, ew, _ = dao.forward(xq.cpu().numpy(), xv.cpu().numpy(), xv.cpu().numpy(), mode, p.get("scale"),
                            p.get("concat_score_weight"), (ids_q != 0).cpu().numpy(), (ids_v != 0).cpu().numpy())
    _check("out", out, eo)
    _check("weights", w, ew)
    assert float(out[0].abs().max()) == 0.0


def test_input_errors():
  q = torch.zeros((2, 3, 129), device="cuda")
  with pytest.raises(ValueError, match="128"):
    Attention()([q, q])
  with pytest.raises(ValueError, match="128"):
    AdditiveAttention()([torch.zeros((2, 3, 8), device="cuda"), torch.zeros((2, 3, 129), device="cuda"),
                         torch.zeros((2, 3, 8), device="cuda")])
  with pytest.raises(ValueError, match="list"):
    Attention()(torch.zeros((2, 3, 8), device="cuda"))
  with pytest.raises((TypeError, ValueError, RuntimeError)):
    Attention()([torch.zeros((2, 3, 8)), torch.zeros((2, 3, 8))])


AUC_FLOOR = 0.344   # half the held-out AUC these seeded runs reached on an H100 (dot 0.6890, concat 0.6885, additive 0.6893)


class _TargetAttentionRanker(tfrs.Model):
  """A DIN-style ranker: the candidate attends over the user's history, then an MLP scores [interest, candidate]."""

  def __init__(self, ids, mode, d=32):
    super().__init__()
    self.lookup = tfrs.layers.StringLookup(vocabulary=ids, mask_token=None)
    self.item = Embedding(len(ids) + 1, d)
    self.attention = _layer_pair(mode, use_scale=True, dropout=0.1, seed=0)
    self.mlp = tfrs.layers.blocks.MLP([64, 1], final_activation="sigmoid")
    self.task = tfrs.tasks.Ranking(metrics=[tfrs.metrics.AUC(name="AUC")])

  def compute_loss(self, inputs, training=False):
    hist = self.item(self.lookup(inputs["history"]))
    cand = self.item(self.lookup(inputs["candidate"]))
    interest = self.attention([cand[:, None, :], hist])[:, 0]
    return self.task(inputs["label"], self.mlp(torch.cat([interest, cand], -1)))


def _ranking_data(n_rows=24576):
  ids, ctx, label = _histories(seed=1, rows=n_rows)
  rng = np.random.RandomState(1)
  neg = ids[rng.randint(0, len(ids), size=n_rows)]
  pos = rng.rand(n_rows) < 0.5
  cand = np.where(pos, label, neg)
  y = torch.from_numpy((pos | (cand == label)).astype(np.float32)[:, None]).cuda()
  return ids, {"history": ctx, "candidate": cand, "label": y}


@pytest.mark.parametrize("mode", dao.MODES)
def test_target_attention_ranker_trains_end_to_end(monkeypatch, mode):
  banned = _ban(monkeypatch, ("scaled_dot_product_attention", "softmax", "multi_head_attention_forward"))
  for name in ("softmax", "bmm", "baddbmm", "matmul", "einsum"):
    monkeypatch.setattr(torch, name, banned)
  ids, data = _ranking_data()
  n_train = 20480
  train = Dataset.from_tensor_slices({k: v[:n_train] for k, v in data.items()}).batch(512)
  test = Dataset.from_tensor_slices({k: v[n_train:] for k, v in data.items()}).batch(2048)
  torch.manual_seed(0)
  model = _TargetAttentionRanker(ids, mode)
  model.compile(optimizer=tfrs.optimizers.Adam(learning_rate=3e-3))
  before = model.evaluate(test)
  hist = model.fit(train, epochs=3)
  after = model.evaluate(test)
  auc = float(after["AUC"])
  print(f"target-attention ranker ({mode}): loss {float(before['loss']):.4f} -> {float(after['loss']):.4f}, "
        f"held-out AUC {float(before['AUC']):.4f} -> {auc:.4f}")
  assert model.attention._calls == 3 * (n_train // 512)
  assert all(np.isfinite(float(h["loss"])) for h in hist)
  assert float(after["loss"]) < float(before["loss"])
  assert auc >= AUC_FLOOR
  assert auc >= float(before["AUC"]) + 0.1, "held-out AUC did not rise: the model learned nothing"
