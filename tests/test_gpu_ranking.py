"""GPU tests of the ranking side (through the C ABI): the Dense layer K6 (tensor-core and exact paths, forward and every
gradient, against the float64 oracle at 1e-5 of each tensor's own scale; the narrow path bit-exact with the canonical fmaf
chain of the C oracle), the cfg5 top stack at full size, `tasks.Ranking` with the fused loss / metrics kernel, and
`experimental.models.Ranking` (mirrors experimental/models/ranking_test.py:115-174 without the TPU size-threshold axis)."""
import itertools
import math
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import ranking_oracle as orc  # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def tfrs():
  import recommenders_b200 as t
  return t


def _rand(shape, seed, scale=1.0):
  g = torch.Generator(device="cuda"); g.manual_seed(seed)
  return torch.randn(shape, generator=g, device="cuda") * scale


def _close(name, got, ref, tol=1e-5):
  got = np.asarray(got.detach().cpu().numpy() if isinstance(got, torch.Tensor) else got, np.float64)
  ref = np.asarray(ref, np.float64)
  err = np.abs(got - ref).max() if ref.size else 0.0
  scale = np.abs(ref).max() if ref.size else 0.0
  assert err <= tol * max(scale, 1e-30), (name, err, scale)


def _act_grad64(act, y, g):
  """dz in float64 from the kernel's own output y (so a relu mask is the kernel's mask)."""
  y = np.asarray(y, np.float64)
  if act == "relu":
    return g * (y > 0)
  if act == "sigmoid":
    return g * y * (1.0 - y)
  return g


# ------------------------------------------------------------------------------------------------
# K6 Dense: forward + dx / dW / db for every activation
# ------------------------------------------------------------------------------------------------
DENSE_SHAPES = [(2048, 256, 512), (1536, 1500, 192), (1500, 845, 130), (3000, 300, 1), (513, 70, 16), (37, 50, 20), (1024, 64, 64)]


@pytest.mark.parametrize("B,K,N", DENSE_SHAPES)
@pytest.mark.parametrize("act", [None, "relu", "sigmoid"])
def test_dense_forward_and_grads_vs_float64(tfrs, B, K, N, act):
  ops = tfrs.ops
  x = _rand((B, K), B + K).requires_grad_(True)
  W = _rand((K, N), N + 7, 1.0 / math.sqrt(K)).requires_grad_(True)
  b = _rand((N,), N + 11, 0.5).requires_grad_(True)
  gy = _rand((B, N), 3)
  y = ops.dense(x, W, b, act)
  y.backward(gy)
  assert ops.dense_uses_tc(B, K, N) == (B >= 1024 and K >= 64 and N >= 64)
  xn, Wn, bn = (t.detach().cpu().numpy() for t in (x, W, b))
  _close("y", y, orc.dense(xn, Wn, bn, act))
  dz = _act_grad64(act, y.detach().cpu().numpy(), gy.cpu().numpy().astype(np.float64))
  _close("dx", x.grad, dz @ Wn.astype(np.float64).T)
  _close("dW", W.grad, xn.astype(np.float64).T @ dz)
  _close("db", b.grad, dz.sum(0))


@pytest.mark.parametrize("B,K,N", [(3000, 300, 1), (513, 70, 16), (37, 50, 20), (100, 1, 3)])
@pytest.mark.parametrize("act", [None, "relu"])
def test_dense_exact_path_bit_exact_with_fmaf_chain(tfrs, B, K, N, act):
  x = _rand((B, K), 5); W = _rand((K, N), 6, 0.1); b = _rand((N,), 7)
  y = tfrs.ops.dense(x, W, b, act)
  ref = orc.dense_chain(x.cpu().numpy(), W.cpu().numpy(), b.cpu().numpy(), act)
  np.testing.assert_array_equal(y.cpu().numpy().view(np.uint32), ref.view(np.uint32))


def test_dense_sigmoid_carries_logits_and_the_loss_uses_them(tfrs):
  """A fused sigmoid output carries its logits; BinaryCrossentropy then takes the logits form (tf-keras `_keras_logits`), and
  the gradient reaches the layer as sigmoid(z) - y per example."""
  B, K = 4000, 96
  x = _rand((B, K), 21); W = (_rand((K, 1), 22, 0.5)).requires_grad_(True); b = torch.zeros(1, device="cuda", requires_grad=True)
  y = (torch.rand((B, 1), device="cuda") > 0.5).float()
  pred = tfrs.ops.dense(x, W, b, "sigmoid")
  z = tfrs.ops.attached_logits(pred)
  assert z is not None and z.shape == pred.shape
  loss = tfrs.losses.BinaryCrossentropy()(y, pred)
  zn = z.detach().cpu().numpy().astype(np.float64)
  exp = orc.ranking_loss(y.cpu().numpy(), zn, from_logits=True)
  assert abs(float(loss.detach()) - exp) <= 1e-5 * abs(exp)
  loss.backward()
  dz = (1.0 / (1.0 + np.exp(-zn)) - y.cpu().numpy()) / B
  _close("db", b.grad, dz.sum(0))
  _close("dW", W.grad, x.cpu().numpy().astype(np.float64).T @ dz)
  # a modified prediction is no longer the layer's output: back to the probability form
  p2 = pred.detach().clone()
  assert tfrs.ops.attached_logits(p2) is None


def test_cfg5_top_stack_full_batch_vs_float64(tfrs):
  """cfg5's top stack at B = 65536: 845 -> 512 (relu) -> 256 (relu) -> 1 (sigmoid), forward + backward.  Each layer is checked
  against float64 from its own input: sampled rows of the outputs and of dx, the whole dW / db."""
  ops = tfrs.ops
  B, dims = 65536, [845, 512, 256, 1]
  acts = ["relu", "relu", "sigmoid"]
  g = torch.Generator(device="cuda"); g.manual_seed(12)
  x = torch.rand((B, dims[0]), generator=g, device="cuda").requires_grad_(True)
  Ws = [(torch.randn((dims[i], dims[i + 1]), generator=g, device="cuda") / math.sqrt(dims[i])).requires_grad_(True) for i in range(3)]
  bs = [(torch.randn((dims[i + 1],), generator=g, device="cuda") * 0.1).requires_grad_(True) for i in range(3)]
  hs = [x]
  for i in range(3):
    h = ops.dense(hs[-1], Ws[i], bs[i], acts[i])
    h.retain_grad()
    hs.append(h)
  gout = torch.randn((B, 1), generator=g, device="cuda")
  hs[-1].backward(gout)
  rows = np.arange(0, B, B // 64)
  for i in range(3):
    hin = hs[i].detach().cpu().numpy().astype(np.float64)
    Wn = Ws[i].detach().cpu().numpy().astype(np.float64); bn = bs[i].detach().cpu().numpy().astype(np.float64)
    hout = hs[i + 1].detach().cpu().numpy()
    _close(f"y{i}", hout[rows], orc.dense(hin[rows], Wn, bn, acts[i]))
    gup = (hs[i + 1].grad if i < 2 else gout).cpu().numpy().astype(np.float64)
    dz = _act_grad64(acts[i], hout, gup)
    _close(f"dx{i}", hs[i].grad[rows], dz[rows] @ Wn.T)
    _close(f"dW{i}", Ws[i].grad, hin.T @ dz)
    _close(f"db{i}", bs[i].grad, dz.sum(0))


# ------------------------------------------------------------------------------------------------
# routing: no torch GEMM / loss on the path
# ------------------------------------------------------------------------------------------------
def _forbid(monkeypatch, target, names):
  for n in names:
    def boom(*a, _n=n, **k):
      raise AssertionError(f"{_n} called on the fused path")
    monkeypatch.setattr(target, n, boom)


def test_mlp_and_ranking_task_stay_on_the_package_kernels(tfrs, monkeypatch):
  mlp = tfrs.layers.blocks.MLP([512, 256, 1], final_activation="sigmoid")
  task = tfrs.tasks.Ranking(metrics=[tfrs.metrics.AUC(), tfrs.metrics.BinaryAccuracy(), tfrs.metrics.RootMeanSquaredError()],
                            prediction_metrics=[tfrs.metrics.Mean("p")], label_metrics=[tfrs.metrics.Mean("l")])
  x = _rand((2048, 845), 1).requires_grad_(True)
  labels = (torch.rand((2048, 1), device="cuda") > 0.5).float()
  assert tfrs.ops.dense_uses_tc(2048, 845, 512) and tfrs.ops.dense_uses_tc(2048, 512, 256)
  _forbid(monkeypatch, tfrs.ops, ["matmul", "sgemm", "gemm_tc"])
  _forbid(monkeypatch, torch, ["matmul", "mm", "addmm"])
  _forbid(monkeypatch, torch.nn.functional, ["linear", "binary_cross_entropy", "binary_cross_entropy_with_logits", "mse_loss"])
  n0 = tfrs.ops.launch_count()
  loss = task(labels, mlp(x), sample_weight=torch.rand(2048, device="cuda"))
  loss.backward()
  assert tfrs.ops.launch_count() > n0
  assert all(l.kernel.grad is not None for l in mlp._sublayers) and x.grad is not None


# ------------------------------------------------------------------------------------------------
# determinism
# ------------------------------------------------------------------------------------------------
def test_two_identical_steps_are_bitwise_equal(tfrs):
  def step():
    torch.manual_seed(3)
    mlp = tfrs.layers.blocks.MLP([512, 256, 1], final_activation="sigmoid")
    mets = [tfrs.metrics.AUC(), tfrs.metrics.BinaryAccuracy(), tfrs.metrics.RootMeanSquaredError()]
    task = tfrs.tasks.Ranking(metrics=mets)
    x = _rand((8192, 845), 2)
    labels = (_rand((8192,), 4) > 0).float()
    w = _rand((8192,), 5).abs()
    loss = task(labels, mlp(x).reshape(-1), sample_weight=w)
    loss.backward()
    grads = [p.grad.clone() for p in mlp.parameters()]
    return float(loss), grads, [m.result() for m in mets]
  l1, g1, m1 = step()
  l2, g2, m2 = step()
  assert l1 == l2 and m1 == m2
  assert all(torch.equal(a, b) for a, b in zip(g1, g2))


# ------------------------------------------------------------------------------------------------
# tasks.Ranking
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("enable_sample_weight", [True, False])
def test_ranking_task_reference_known_answers(tfrs, enable_sample_weight):
  """tasks/ranking_test.py:29-62."""
  task = tfrs.tasks.Ranking(metrics=[tfrs.metrics.BinaryAccuracy(name="accuracy")],
                            label_metrics=[tfrs.metrics.Mean(name="label_mean")],
                            prediction_metrics=[tfrs.metrics.Mean(name="prediction_mean")],
                            loss_metrics=[tfrs.metrics.Mean(name="loss_mean")])
  predictions = torch.tensor([[1.0], [0.3]], device="cuda")
  labels = torch.tensor([[1.0], [1.0]], device="cuda")
  sample_weight = torch.tensor([1.0, 1.0], device="cuda") if enable_sample_weight else None
  expected_loss = -(math.log(1) + math.log(0.3)) / 2.0
  expected = {"accuracy": 0.5, "label_mean": 1.0, "prediction_mean": 0.65, "loss_mean": expected_loss}
  loss = task(predictions=predictions, labels=labels, sample_weight=sample_weight)
  got = {m.name: m.result() for m in task.metrics}
  assert float(loss) == pytest.approx(expected_loss, rel=1e-6, abs=1e-6)
  assert set(got) == set(expected)
  for k, v in expected.items():
    assert got[k] == pytest.approx(v, rel=1e-6, abs=1e-6), k
  # compute_metrics=False leaves the metrics untouched
  task(predictions=predictions, labels=labels, compute_metrics=False)
  assert {m.name: m.result() for m in task.metrics} == got


@pytest.mark.parametrize("weighted", [False, True])
@pytest.mark.parametrize("loss_name", ["bce", "bce_logits", "mse"])
def test_ranking_task_matches_oracle_on_100k_rows(tfrs, weighted, loss_name):
  B = 100_000
  rng = np.random.RandomState(7)
  p = rng.rand(B).astype(np.float32)
  p[:50] = 0.0; p[50:100] = 1.0; p[100:150] = 0.5      # bucket edges and the clip
  y = (rng.rand(B) < p).astype(np.float32)
  w = rng.rand(B).astype(np.float32) if weighted else None
  loss_obj = {"bce": tfrs.losses.BinaryCrossentropy(), "bce_logits": tfrs.losses.BinaryCrossentropy(from_logits=True),
              "mse": tfrs.losses.MeanSquaredError()}[loss_name]
  pin = (p * 8 - 4) if loss_name == "bce_logits" else p
  auc, acc, rmse = tfrs.metrics.AUC(), tfrs.metrics.BinaryAccuracy(), tfrs.metrics.RootMeanSquaredError()
  mse = tfrs.metrics.MeanSquaredError()
  pm, lm, lossm = tfrs.metrics.Mean("p"), tfrs.metrics.Mean("l"), tfrs.metrics.Mean("loss")
  task = tfrs.tasks.Ranking(loss=loss_obj, metrics=[auc, acc, rmse, mse], prediction_metrics=[pm], label_metrics=[lm],
                            loss_metrics=[lossm])
  pt = torch.from_numpy(pin).cuda().reshape(B, 1).requires_grad_(True)
  yt = torch.from_numpy(y).cuda().reshape(B, 1)
  wt = None if w is None else torch.from_numpy(w).cuda()
  loss = task(yt, pt, sample_weight=wt)
  kind = "mse" if loss_name == "mse" else "bce"
  exp = orc.ranking_loss(y, pin, w, loss=kind, from_logits=loss_name == "bce_logits")
  assert abs(float(loss) - exp) <= 1e-5 * abs(exp), (float(loss), exp)
  assert lossm.result() == pytest.approx(float(loss), rel=1e-7)
  assert acc.result() == pytest.approx(orc.binary_accuracy(y, pin, w), rel=1e-9, abs=1e-12)
  assert rmse.result() == pytest.approx(orc.rmse(y, pin, w), rel=1e-9)
  assert mse.result() == pytest.approx(orc.rmse(y, pin, w) ** 2, rel=1e-9)
  assert pm.result() == pytest.approx(orc.weighted_mean(pin, w), rel=1e-9)
  assert lm.result() == pytest.approx(orc.weighted_mean(y, w), rel=1e-9)
  pos, neg = orc.auc_buckets(y, pin, w)
  gpos, gneg = auc.bucket_counts()
  if w is None:
    np.testing.assert_array_equal(gpos, pos); np.testing.assert_array_equal(gneg, neg)
  else:
    np.testing.assert_allclose(gpos, pos, rtol=1e-9); np.testing.assert_allclose(gneg, neg, rtol=1e-9)
  assert auc.result() == pytest.approx(orc.auc(y, pin, w), rel=1e-9, abs=1e-12)
  # gradient of the loss w.r.t. the predictions (the logits for from_logits)
  loss.backward()
  x64 = pin.astype(np.float64); y64 = y.astype(np.float64); w64 = np.ones(B) if w is None else w.astype(np.float64)
  if loss_name == "mse":
    d = 2 * (x64 - y64)
  elif loss_name == "bce_logits":
    d = 1 / (1 + np.exp(-x64)) - y64
  else:
    eps = float(np.float32(1e-7))
    inside = (x64 >= eps) & (x64 <= 1 - eps)
    d = np.where(inside, -y64 / (x64 + eps) + (1 - y64) / (1 - x64 + eps), 0.0)
  _close("dpred", pt.grad.reshape(-1), d * w64 / B)
  # reset
  for m in task.metrics:
    m.reset_states()
  assert acc.result() == 0.0 and auc.result() == 0.0


def test_ranking_task_reductions_and_custom_objects(tfrs):
  B = 3000
  rng = np.random.RandomState(3)
  p = rng.rand(B).astype(np.float32); y = (rng.rand(B) > 0.5).astype(np.float32); w = rng.rand(B).astype(np.float32)
  pt, yt, wt = (torch.from_numpy(a).cuda() for a in (p, y, w))
  for red in ("none", "sum", "sum_over_batch_size"):
    loss = tfrs.losses.BinaryCrossentropy(reduction=red)(yt, pt, sample_weight=wt)
    exp = orc.ranking_loss(y, p, w, reduction=red)
    _close(red, loss, exp)
    assert (loss.shape == (B,)) == (red == "none")

  class Custom:          # any object with update_state is called as is
    name = "custom"
    def __init__(self): self.calls = 0
    def update_state(self, y_true=None, y_pred=None, sample_weight=None): self.calls += 1
    def reset_states(self): self.calls = 0
    def result(self): return self.calls
  c = Custom()
  task = tfrs.tasks.Ranking(loss=lambda y_true, y_pred, sample_weight=None: ((y_pred - y_true) ** 2).mean(), metrics=[c, tfrs.metrics.AUC()])
  task(yt, pt)
  assert c.calls == 1 and task.metrics[1].result() == pytest.approx(orc.auc(y, p), rel=1e-9)
  with pytest.raises(NotImplementedError):
    tfrs.metrics.AUC(curve="PR")


# ------------------------------------------------------------------------------------------------
# experimental.models.Ranking  (experimental/models/ranking_test.py:115-174, without the TPU size_threshold axis)
# ------------------------------------------------------------------------------------------------
def _synthetic_data(num_dense, vocab_sizes, dataset_size, batch_size, generate_weights, seed=0):
  """experimental/models/ranking_test.py:_generate_synthetic_data: labels = int((mean(dense) + sum(ids)/sum(vocab)) / 2 + 0.5)."""
  g = torch.Generator(device="cuda"); g.manual_seed(seed)
  dense = torch.rand((dataset_size, num_dense), generator=g, device="cuda")
  sparse = [torch.randint(0, v, (dataset_size,), generator=g, device="cuda", dtype=torch.int32) for v in vocab_sizes]
  sparse_mean = torch.stack(sparse, -1).sum(1).float() / sum(vocab_sizes)
  labels = ((dense.mean(1) + sparse_mean) / 2.0 + 0.5).to(torch.int32)
  weights = torch.rand((dataset_size, 1), generator=g, device="cuda") if generate_weights else None
  batches = []
  for lo in range(0, dataset_size - batch_size + 1, batch_size):
    feats = {"dense_features": dense[lo:lo + batch_size], "sparse_features": {str(i): s[lo:lo + batch_size] for i, s in enumerate(sparse)}}
    batches.append((feats, labels[lo:lo + batch_size]) if weights is None else (feats, labels[lo:lo + batch_size], weights[lo:lo + batch_size]))
  return batches


def _embedding(tfrs, vocab_sizes, dim=16):
  return torch.nn.ModuleDict({str(i): tfrs.layers.embedding.Embedding(v, dim) for i, v in enumerate(vocab_sizes)})


class _ConcatCross(torch.nn.Module):
  """tf.keras.Sequential([Concatenate(), Cross()])."""

  def __init__(self, tfrs):
    super().__init__()
    self.cross = tfrs.layers.feature_interaction.Cross()

  def forward(self, inputs):
    return self.cross(torch.cat(inputs, dim=1))


@pytest.mark.parametrize("interaction,bottom,top,concat_dense,use_weights",
                         list(itertools.product(("dot", "cross"), ("default", "mlp"), ("default", "mlp"), (True, False), (True, False))))
def test_ranking_model(tfrs, interaction, bottom, top, concat_dense, use_weights):
  vocab = [30, 3, 26]
  torch.manual_seed(0)
  model = tfrs.experimental.models.Ranking(
      embedding_layer=_embedding(tfrs, vocab),
      bottom_stack=None if bottom == "default" else tfrs.layers.blocks.MLP(units=[40, 16]),
      feature_interaction=tfrs.layers.feature_interaction.DotInteraction() if interaction == "dot" else _ConcatCross(tfrs),
      top_stack=None if top == "default" else tfrs.layers.blocks.MLP(units=[40, 20, 1], final_activation="sigmoid"),
      concat_dense=concat_dense)
  model.compile(optimizer=tfrs.optimizers.Adagrad(0.1))
  data = _synthetic_data(8, vocab, 64, 16, use_weights)
  history = model.fit([data[i % len(data)] for i in range(5)], epochs=1)
  assert np.isfinite(float(history[-1]["loss"]))
  metrics = model.evaluate(data, return_dict=True)
  assert "loss" in metrics and "accuracy" in metrics
  assert 0.0 <= metrics["accuracy"] <= 1.0 and np.isfinite(float(metrics["loss"]))
  assert len(model.dense_trainable_variables) > 0 and len(model.embedding_trainable_variables) == 3


def test_ranking_model_input_errors_and_loss_decreases(tfrs):
  vocab = [30, 3, 26]
  torch.manual_seed(1)
  model = tfrs.experimental.models.Ranking(embedding_layer=_embedding(tfrs, vocab))
  data = _synthetic_data(8, vocab, 64, 16, False, seed=5)
  with pytest.raises(ValueError, match="Inputs should be either a tuple of"):
    model.compute_loss((data[0][0],))
  model.compile(optimizer=tfrs.optimizers.Adagrad(0.05))
  losses = []
  for _ in range(15):
    hist = model.fit(data, epochs=1)
    losses.append(float(model.evaluate(data)["loss"]))
  assert losses[-1] < losses[0], losses
  m = model.evaluate(data)
  assert {"auc", "accuracy", "prediction_mean", "label_mean", "loss"} <= set(m)
