"""The dense attention oracle (tests/dense_attention_oracle.py) against float64 torch autograd and central differences,
and the host side of layers.Attention / layers.AdditiveAttention: constructor checks, configs, weights, seeds, the ABI."""
import math
import os
import re

import numpy as np
import pytest
import torch

import dense_attention_oracle as dao
import regularization_oracle as ro
from recommenders_b200.layers import AdditiveAttention, Attention


def _torch_forward(q, k, v, mode, scale, wc, qm, vm, causal, drop_keep, rate):
  B, Tq, _ = q.shape
  Tv = k.shape[1]
  if mode == "dot":
    s = q @ k.transpose(1, 2)
    s = s if scale is None else s * scale
  else:
    u = q[:, :, None, :] + k[:, None, :, :]
    if mode == "concat":
      s = wc * torch.tanh(u if scale is None else scale * u).sum(-1)
    else:
      t = torch.tanh(u)
      s = t.sum(-1) if scale is None else (t * scale).sum(-1)
  keep = torch.from_numpy(dao.keep_mask(B, Tq, Tv, vm, causal))
  m = s - 1e9
  s = torch.where(keep, s, m + (m.float().double() - m).detach())   # the fp32 value, a float64 gradient
  w = torch.softmax(s, -1)
  if drop_keep is not None:
    w = torch.where(torch.from_numpy(drop_keep), w / (1 - rate), torch.zeros_like(w))
  out = w @ v
  if qm is not None:
    out = out * torch.from_numpy(qm.astype(np.float64))[..., None]
  return out, w


CASES = [(mode, use_scale, masked, causal, rate) for mode in dao.MODES for use_scale in (False, True)
         for masked, causal, rate in ((False, False, 0.0), (True, False, 0.0), (True, True, 0.0), (True, True, 0.3),
                                      (False, False, 0.5))]


@pytest.mark.parametrize("mode,use_scale,masked,causal,rate", CASES)
def test_oracle_matches_float64_autograd(mode, use_scale, masked, causal, rate):
  rng = np.random.RandomState(7)
  B, Tq, Tv, dim, dv = 3, 5, 6, 4, 3
  q, k, v = rng.normal(size=(B, Tq, dim)), rng.normal(size=(B, Tv, dim)), rng.normal(size=(B, Tv, dv))
  scale = None
  if use_scale:
    scale = rng.uniform(0.5, 1.5, size=(dim,)) if mode == "additive" else np.float64(1.3)
  wc = 0.8 if mode == "concat" else None
  qm = rng.rand(B, Tq) < 0.7 if masked else None
  vm = rng.rand(B, Tv) < 0.7 if masked else None
  if masked:
    vm[0] = False                                   # a fully masked value row: uniform weights
  drop_keep = ro.dropout_keep((B, Tq, Tv), rate, 11, 2) if rate else None
  out, wd, cache = dao.forward(q, k, v, mode, scale, wc, qm, vm, causal, drop_keep, rate)
  g = rng.normal(size=out.shape)
  dq, dk, dv_, dscale, dwc = dao.backward(cache, g)

  tq, tk, tv = (torch.tensor(a, requires_grad=True) for a in (q, k, v))
  ts = None if scale is None else torch.tensor(scale, requires_grad=True)
  tw = None if wc is None else torch.tensor(wc, dtype=torch.float64, requires_grad=True)
  tout, tw_ = _torch_forward(tq, tk, tv, mode, ts, tw, qm, vm, causal, drop_keep, rate)
  tout.backward(torch.from_numpy(g))
  np.testing.assert_allclose(out, tout.detach().numpy(), rtol=1e-10, atol=1e-12)
  np.testing.assert_allclose(wd, tw_.detach().numpy(), rtol=1e-10, atol=1e-12)
  for got, t in ((dq, tq), (dk, tk), (dv_, tv), (dscale, ts), (dwc, tw)):
    if t is None:
      assert got is None
    else:
      np.testing.assert_allclose(got, t.grad.numpy(), rtol=1e-9, atol=1e-11)


@pytest.mark.parametrize("mode", dao.MODES)
def test_oracle_matches_central_differences(mode):
  """A masked, causal, dropped-out case: every input and weight gradient against central differences of the forward."""
  rng = np.random.RandomState(3)
  B, Tq, Tv, dim, dv = 2, 4, 4, 3, 2
  x = {"q": rng.normal(size=(B, Tq, dim)), "k": rng.normal(size=(B, Tv, dim)), "v": rng.normal(size=(B, Tv, dv)),
       "scale": rng.uniform(0.5, 1.5, size=(dim,)) if mode == "additive" else np.array(1.2),
       "wc": np.array(0.7)}
  qm = np.array([[1, 1, 0, 1], [1, 0, 1, 1]], bool)
  vm = np.array([[1, 0, 1, 1], [1, 1, 1, 0]], bool)
  rate = 0.25
  keep = ro.dropout_keep((B, Tq, Tv), rate, 5, 1)
  g = rng.normal(size=(B, Tq, dv))

  def loss(p):
    out, _, _ = dao.forward(p["q"], p["k"], p["v"], mode, p["scale"], p["wc"] if mode == "concat" else None, qm, vm,
                            True, keep, rate)
    return float((out * g).sum())

  _, _, cache = dao.forward(x["q"], x["k"], x["v"], mode, x["scale"], x["wc"] if mode == "concat" else None, qm, vm,
                            True, keep, rate)
  dq, dk, dv_, dscale, dwc = dao.backward(cache, g)
  grads = {"q": dq, "k": dk, "v": dv_, "scale": dscale}
  if mode == "concat":
    grads["wc"] = dwc
  h = 1e-6
  for name, an in grads.items():
    num = np.zeros_like(x[name], dtype=np.float64)
    for idx in np.ndindex(*x[name].shape):
      p = {n: a.copy() for n, a in x.items()}
      p[name][idx] += h
      up = loss(p)
      p[name][idx] -= 2 * h
      num[idx] = (up - loss(p)) / (2 * h)
    np.testing.assert_allclose(np.asarray(an).reshape(num.shape), num, rtol=1e-5, atol=1e-7, err_msg=name)


def test_constructor_checks():
  with pytest.raises(ValueError, match="score_mode"):
    Attention(score_mode="general")
  for cls in (Attention, AdditiveAttention):
    with pytest.raises(TypeError, match="use_scael"):
      cls(use_scael=True)
    with pytest.raises(NotImplementedError, match="dtype"):
      cls(dtype="float16")
    with pytest.raises(NotImplementedError, match="trainable"):
      cls(trainable=False)
    cls(dtype="float32", trainable=True)
  for rate in (-0.1, 1.0, 1.5):
    with pytest.raises(ValueError, match="dropout"):
      Attention(dropout=rate)
    with pytest.raises(ValueError, match="dropout"):
      AdditiveAttention(dropout=rate)


@pytest.mark.parametrize("layer", [Attention(), Attention(use_scale=True, score_mode="concat", dropout=0.2, seed=3),
                                   Attention(causal=True, name="att"), AdditiveAttention(),
                                   AdditiveAttention(use_scale=False, dropout=0.1, seed=9, name="add")])
def test_configs_round_trip(layer):
  cfg = layer.get_config()
  again = type(layer).from_config(cfg)
  assert again.get_config() == cfg
  assert again._key == layer._key and again.causal == layer.causal


def test_weights_names_shapes_and_initialisers():
  cpu = torch.device("cpu")
  a = Attention(use_scale=True, score_mode="concat")
  a.build(16, cpu)
  assert sorted(n for n, _ in a.named_parameters()) == ["concat_score_weight", "scale"]
  for p in (a.scale, a.concat_score_weight):
    assert p.shape == () and float(p.detach()) == 1.0
  b = Attention()
  b.build(16, cpu)
  assert list(b.named_parameters()) == []
  c = Attention(score_mode="concat")
  c.build(16, cpu)
  assert [n for n, _ in c.named_parameters()] == ["concat_score_weight"]
  torch.manual_seed(0)
  d = AdditiveAttention()
  d.build(300, cpu)
  assert [n for n, _ in d.named_parameters()] == ["scale"] and d.scale.shape == (300,)
  limit = math.sqrt(6.0 / (300 + 300))                # Keras's fans of a 1-D weight: (dim, dim)
  s = d.scale.detach().numpy()
  assert np.abs(s).max() <= limit and np.abs(s).max() > 0.9 * limit and abs(s.mean()) < 0.2 * limit
  e = AdditiveAttention(use_scale=False)
  e.build(8, cpu)
  assert list(e.named_parameters()) == []


def test_seed_handling():
  state = torch.get_rng_state()
  Attention(score_mode="concat")
  AdditiveAttention(dropout=0.0)
  Attention(dropout=0.5, seed=4)
  assert torch.equal(state, torch.get_rng_state()), "a layer without a drawn key moved torch's RNG"
  torch.manual_seed(1)
  k1 = Attention(dropout=0.1)._key
  torch.manual_seed(1)
  assert AdditiveAttention(dropout=0.1)._key == k1
  assert Attention(dropout=0.1, seed=2**64 + 5)._key == 5


def test_abi_names_are_declared():
  header = open(os.path.join(os.path.dirname(__file__), "..", "include", "tfrs_b200.h")).read()
  for name in ("tfrs_dense_attention_fwd_f32", "tfrs_dense_attention_bwd_workspace_bytes",
               "tfrs_dense_attention_bwd_f32"):
    assert re.search(r"\b" + name + r"\(", header), name
  for name in ("TFRS_DENSE_DOT 0", "TFRS_DENSE_CONCAT 1", "TFRS_DENSE_ADDITIVE 2", "TfrsDenseAttention"):
    assert name in header


@pytest.mark.parametrize("mode", ["dot", "concat"])
def test_weight_grad_rows_sum_to_the_weight_gradients(mode):
  rng = np.random.RandomState(1)
  q, k = rng.normal(size=(2, 3, 4)), rng.normal(size=(2, 5, 4))
  v, g = rng.normal(size=(2, 5, 2)), rng.normal(size=(2, 3, 2))
  _, _, cache = dao.forward(q, k, v, mode, 1.1, 0.9 if mode == "concat" else None, value_mask=rng.rand(2, 5) < 0.7,
                            drop_keep=ro.dropout_keep((2, 3, 5), 0.2, 1, 0), rate=0.2)
  _, _, _, dscale, dwc = dao.backward(cache, g)
  rs, rw = dao.weight_grad_rows(cache, g)
  np.testing.assert_allclose(rs.sum(), dscale, rtol=1e-12)
  if mode == "concat":
    np.testing.assert_allclose(rw.sum(), dwc, rtol=1e-12)
  else:
    assert rw is None
