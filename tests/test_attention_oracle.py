"""CPU tests of the MultiHeadAttention and LayerNormalization rules: the float64 oracle (tests/attention_oracle.py)
against float64 torch (SDPA with the additive mask, layer_norm, autograd for every gradient) and against central
differences on a masked causal case; fully masked rows; Keras's fans in the initializer; constructor errors; config
round trips; and the ABI declarations of K21 / K22."""
import os
import re

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import attention_oracle as ao
from recommenders_b200 import ops
from recommenders_b200.layers import LayerNormalization, MultiHeadAttention
from recommenders_b200.layers.attention import keras_fans

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _weights(rng, Dq, Dk, Dv, H, dk, dv, Dout, bias=True):
  w = lambda *s: rng.uniform(-0.5, 0.5, size=s)
  W = (w(Dq, H, dk), w(Dk, H, dk), w(Dv, H, dv), w(H, dv, Dout))
  b = (w(H, dk) * 0.2, w(H, dk) * 0.2, w(H, dv) * 0.2, w(Dout) * 0.2) if bias else (None,) * 4
  return W, b


def _torch_mha(query, value, key, W, b, keep):
  """float64 torch: the projections, Q scaled by float32(1/sqrt(dk)), SDPA with the additive -1e9 mask, the output
  projection.  Every tensor requires grad."""
  B, T, _ = query.shape
  S = value.shape[1]
  H, dk, dv = W[0].shape[1], W[0].shape[2], W[2].shape[2]
  proj = lambda x, Wt, bt: x @ Wt.reshape(Wt.shape[0], -1) + (0 if bt is None else bt.reshape(-1))
  Q = proj(query, W[0], b[0]).reshape(B, T, H, dk).transpose(1, 2) * ao.scale_of(dk)
  K = proj(key, W[1], b[1]).reshape(B, S, H, dk).transpose(1, 2)
  V = proj(value, W[2], b[2]).reshape(B, S, H, dv).transpose(1, 2)
  add = None if keep is None else torch.where(torch.from_numpy(np.array(keep))[:, None], 0.0, ao.MASK_ADDER)
  O = F.scaled_dot_product_attention(Q, K, V, attn_mask=add, scale=1.0)
  out = O.transpose(1, 2).reshape(B, T, H * dv) @ W[3].reshape(H * dv, -1)
  return out if b[3] is None else out + b[3]


CASES = [  # B, T, S, Dq, Dv, Dk (None: key = value), H, dk, dv, Dout, bias, masks
    (2, 5, 5, 6, 6, None, 2, 3, 3, 6, True, "causal"),
    (3, 4, 7, 5, 3, 4, 1, 2, 5, 4, True, "value+query"),
    (2, 6, 3, 4, 4, None, 3, 4, 2, 7, False, "attention+key"),
    (1, 1, 1, 2, 2, 3, 1, 1, 1, 2, True, None),
]


def _keep(kind, B, T, S, rng):
  """A combined mask with no fully masked row (the additive mask in float64 is not rounded to float32, so such a row
  would differ from Keras's)."""
  if kind is None:
    return None, {}
  m = {}
  if "causal" in kind:
    m["causal"] = True
  if "value" in kind:
    v = rng.rand(B, S) < 0.6
    v[:, 0] = True
    m["value_mask"] = v
  if "key" in kind:
    k = rng.rand(B, S) < 0.7
    k[:, -1] = True
    m["key_mask"] = k
  if "attention" in kind:
    a = rng.rand(B, T, S) < 0.6
    a[:, :, -1] = True
    m["attention_mask"] = a
  keep = ao.combined_mask(B, T, S, **m)
  if "query" in kind:       # a masked query row is fully masked: checked in its own test
    m["query_mask"] = np.ones((B, T), bool)
  return ao.combined_mask(B, T, S, **m), m


@pytest.mark.parametrize("case", CASES)
def test_mha_oracle_matches_float64_torch_forward_and_gradients(case):
  B, T, S, Dq, Dv, Dk, H, dk, dv, Dout, bias, masks = case
  rng = np.random.RandomState(B * 100 + T * 10 + S)
  W, b = _weights(rng, Dq, Dk or Dv, Dv, H, dk, dv, Dout, bias)
  query, value = rng.normal(size=(B, T, Dq)), rng.normal(size=(B, S, Dv))
  key = None if Dk is None else rng.normal(size=(B, S, Dk))
  keep, _ = _keep(masks, B, T, S, rng)
  g = rng.normal(size=(B, T, Dout))

  tt = lambda a: None if a is None else torch.from_numpy(np.array(a)).requires_grad_()
  qt, vt, kt = tt(query), tt(value), tt(key)
  Wt, bt = [tt(w) for w in W], [tt(x) for x in b]
  out_t = _torch_mha(qt, vt, vt if kt is None else kt, Wt, bt, keep)
  (out_t * torch.from_numpy(g)).sum().backward()

  out, P, cache = ao.mha_forward(query, value, key, *W, *b, keep=keep)
  np.testing.assert_allclose(out, out_t.detach().numpy(), rtol=1e-11, atol=1e-12)
  assert np.allclose(P.sum(-1), 1.0)
  r = ao.mha_backward(cache, g, key_is_value=key is None)
  close = lambda a, e, n: np.testing.assert_allclose(a, e, rtol=1e-9, atol=1e-11, err_msg=n)
  close(r["dquery"], qt.grad.numpy(), "dquery")
  close(r["dvalue"], vt.grad.numpy(), "dvalue")
  if key is not None:
    close(r["dkey"], kt.grad.numpy(), "dkey")
  for i, n in enumerate("qkvo"):
    close(r["dW" + n], Wt[i].grad.numpy(), "dW" + n)
    if bias:
      close(r["db" + n], bt[i].grad.numpy(), "db" + n)


def test_mha_oracle_gradients_match_central_differences_on_a_masked_causal_case():
  rng = np.random.RandomState(5)
  B, T, S, D, H, dk, dv, Dout = 2, 4, 4, 3, 2, 2, 3, 3
  W, b = _weights(rng, D, D, D, H, dk, dv, Dout)
  query, value, key = rng.normal(size=(B, T, D)), rng.normal(size=(B, S, D)), rng.normal(size=(B, S, D))
  vm = np.array([[1, 0, 1, 1], [1, 1, 0, 1]], bool)
  keep = ao.combined_mask(B, T, S, value_mask=vm, causal=True)
  assert keep.any(-1).all()
  g = rng.normal(size=(B, T, Dout))
  args = {"dquery": query, "dvalue": value, "dkey": key, "dWq": W[0], "dWk": W[1], "dWv": W[2], "dWo": W[3],
          "dbq": b[0], "dbk": b[1], "dbv": b[2], "dbo": b[3]}

  def loss():
    out, _, _ = ao.mha_forward(query, value, key, *W, *b, keep=keep)
    return float((out * g).sum())

  r = ao.mha_backward(ao.mha_forward(query, value, key, *W, *b, keep=keep)[2], g)
  eps = 1e-6
  for name, a in args.items():
    num = np.zeros_like(a)
    for idx in np.ndindex(a.shape):
      v0 = a[idx]
      a[idx] = v0 + eps; lp = loss()
      a[idx] = v0 - eps; lm = loss()
      a[idx] = v0
      num[idx] = (lp - lm) / (2 * eps)
    np.testing.assert_allclose(r[name], num, rtol=1e-6, atol=1e-8, err_msg=name)


def test_fully_masked_rows_attend_uniformly():
  rng = np.random.RandomState(2)
  B, T, S, H, dk = 2, 3, 5, 2, 4
  Q, K, V = rng.normal(size=(B, T, H, dk)), rng.normal(size=(B, S, H, dk)), rng.normal(size=(B, S, H, dk))
  qm = np.array([[1, 0, 1], [0, 1, 1]], bool)
  keep = ao.combined_mask(B, T, S, query_mask=qm, causal=True)
  O, P, _ = ao.core_forward(Q, K, V, keep)
  assert np.array_equal(P[0, :, 1], np.full((H, S), 1.0 / S))
  assert np.array_equal(P[1, :, 0], np.full((H, S), 1.0 / S))
  np.testing.assert_allclose(O[0, 1], V[0].mean(0), rtol=1e-12)
  assert not P[0, :, 0, 1:].any()                       # causal: row 0 keeps key 0 alone
  assert np.array_equal(ao.combined_mask(1, 2, 2, causal=True)[0], [[True, False], [True, True]])


@pytest.mark.parametrize("shape", [(4, 7), (2, 3, 1), (3, 2, 33)])
@pytest.mark.parametrize("affine", [True, False])
def test_layer_norm_oracle_matches_float64_torch(shape, affine):
  rng = np.random.RandomState(len(shape) * 10 + shape[-1])
  x = rng.normal(size=shape) * 3 + 2
  d = shape[-1]
  gamma, beta = (rng.normal(size=d), rng.normal(size=d)) if affine else (None, None)
  g = rng.normal(size=shape)
  tt = lambda a: None if a is None else torch.from_numpy(np.array(a)).requires_grad_()
  xt, gt, bt = tt(x), tt(gamma), tt(beta)
  yt = F.layer_norm(xt, (d,), gt, bt, eps=1e-3)
  (yt * torch.from_numpy(g)).sum().backward()
  y, _, _ = ao.layer_norm_forward(x, gamma, beta)
  np.testing.assert_allclose(y, yt.detach().numpy(), rtol=1e-12, atol=1e-12)
  dx, dg, db = ao.layer_norm_backward(x, gamma, g)
  np.testing.assert_allclose(dx, xt.grad.numpy(), rtol=1e-9, atol=1e-11)
  if affine:
    np.testing.assert_allclose(dg, gt.grad.numpy(), rtol=1e-10, atol=1e-12)
    np.testing.assert_allclose(db, bt.grad.numpy(), rtol=1e-10, atol=1e-12)


def test_layer_norm_oracle_gradients_match_central_differences():
  rng = np.random.RandomState(9)
  x, gamma, beta, g = rng.normal(size=(3, 5)), rng.normal(size=5), rng.normal(size=5), rng.normal(size=(3, 5))
  dx, dg, db = ao.layer_norm_backward(x, gamma, g)
  eps = 1e-6
  for got, a in ((dx, x), (dg, gamma), (db, beta)):
    num = np.zeros_like(a)
    for idx in np.ndindex(a.shape):
      v0 = a[idx]
      a[idx] = v0 + eps; lp = (ao.layer_norm_forward(x, gamma, beta)[0] * g).sum()
      a[idx] = v0 - eps; lm = (ao.layer_norm_forward(x, gamma, beta)[0] * g).sum()
      a[idx] = v0
      num[idx] = (lp - lm) / (2 * eps)
    np.testing.assert_allclose(got, num, rtol=1e-6, atol=1e-8)


def test_keras_fans_and_the_glorot_limit():
  assert keras_fans((32, 2, 16)) == (64, 512)            # query kernel [D, H, dk]
  assert keras_fans((2, 16, 32)) == (32, 64)             # output kernel [H, dv, D_out]
  assert keras_fans((5, 7)) == (5, 7) and keras_fans((4,)) == (4, 4)
  torch.manual_seed(0)
  layer = MultiHeadAttention(2, 16)
  layer.build((3, 10, 32), (3, 10, 32), device="cpu")
  for w, shape in ((layer.query.kernel, (32, 2, 16)), (layer.key.kernel, (32, 2, 16)),
                   (layer.value.kernel, (32, 2, 16)), (layer.attention_output.kernel, (2, 16, 32))):
    assert tuple(w.shape) == shape
    fan_in, fan_out = keras_fans(shape)
    limit = np.sqrt(6.0 / (fan_in + fan_out))
    a = w.detach().abs()
    assert a.max() <= limit and a.max() > 0.9 * limit   # uniform on [-limit, limit]
  assert tuple(layer.query.bias.shape) == (2, 16) and tuple(layer.attention_output.bias.shape) == (32,)
  assert not layer.query.bias.any()
  names = {n for n, _ in layer.named_parameters()}
  assert names == {f"{p}.{w}" for p in ("query", "key", "value", "attention_output") for w in ("kernel", "bias")}


def test_shapes_with_value_dim_output_shape_and_no_bias():
  layer = MultiHeadAttention(4, 8, value_dim=5, output_shape=12, use_bias=False)
  layer.build((2, 3, 6), (2, 4, 7), (2, 4, 9), device="cpu")
  assert tuple(layer.query.kernel.shape) == (6, 4, 8) and tuple(layer.key.kernel.shape) == (9, 4, 8)
  assert tuple(layer.value.kernel.shape) == (7, 4, 5) and tuple(layer.attention_output.kernel.shape) == (4, 5, 12)
  assert layer.query.bias is None and layer.attention_output.bias is None


@pytest.mark.parametrize("kwargs,arg", [
    ({"attention_axes": (1, 2)}, "attention_axes"), ({"attention_axes": 2}, "attention_axes"),
    ({"dropout": 0.1}, "dropout"), ({"kernel_regularizer": "l2"}, "kernel_regularizer"),
    ({"bias_regularizer": "l2"}, "bias_regularizer"), ({"activity_regularizer": "l2"}, "activity_regularizer"),
    ({"kernel_constraint": "non_neg"}, "kernel_constraint"), ({"bias_constraint": "non_neg"}, "bias_constraint"),
    ({"output_shape": (4, 5)}, "output_shape")])
def test_mha_unsupported_arguments_raise_naming_the_argument(kwargs, arg):
  with pytest.raises(NotImplementedError, match=arg):
    MultiHeadAttention(2, 8, **kwargs)


def test_mha_head_dims_are_validated_against_the_ceiling():
  MultiHeadAttention(1, ops.MHA_MAX_HEAD_DIM, value_dim=ops.MHA_MAX_HEAD_DIM)
  for kw in ({"key_dim": ops.MHA_MAX_HEAD_DIM + 1}, {"key_dim": 8, "value_dim": ops.MHA_MAX_HEAD_DIM + 1}):
    with pytest.raises(ValueError, match=str(ops.MHA_MAX_HEAD_DIM)):
      MultiHeadAttention(2, **kw)
  for bad in (0, -1, 2.5, True):
    with pytest.raises(ValueError):
      MultiHeadAttention(bad, 8)
  for axes in (None, 1, (1,), [1]):
    MultiHeadAttention(2, 8, attention_axes=axes)


def test_rank_other_than_three_raises():
  layer = MultiHeadAttention(2, 4)
  with pytest.raises(NotImplementedError, match="rank"):
    layer(torch.zeros((2, 3, 4, 5)), torch.zeros((2, 3, 4, 5)))
  with pytest.raises(NotImplementedError, match="rank"):
    layer(torch.zeros((2, 3)), torch.zeros((2, 3)))


def test_layer_norm_unsupported_arguments_raise():
  for kw, arg in (({"beta_regularizer": "l2"}, "beta_regularizer"), ({"gamma_constraint": "x"}, "gamma_constraint"),
                  ({"axis": [1, 2]}, "axis")):
    with pytest.raises(NotImplementedError, match=arg):
      LayerNormalization(**kw)
  ln = LayerNormalization(axis=1)
  with pytest.raises(NotImplementedError, match="axis"):
    ln.build((2, 3, 4), device="cpu")
  LayerNormalization(axis=2).build((2, 3, 4), device="cpu")
  LayerNormalization(axis=[-1]).build((2, 3, 4), device="cpu")


def test_layer_norm_build_and_flags():
  ln = LayerNormalization(center=False)
  ln.build((3, 7), device="cpu")
  assert ln.beta is None and torch.equal(ln.gamma.detach(), torch.ones(7))
  ln = LayerNormalization(scale=False, beta_initializer="ones")
  ln.build((3, 7), device="cpu")
  assert ln.gamma is None and torch.equal(ln.beta.detach(), torch.ones(7))


def test_get_config_round_trips():
  layer = MultiHeadAttention(3, 16, value_dim=8, use_bias=False, output_shape=20, attention_axes=(1,), name="mha",
                             kernel_initializer="truncated_normal")
  cfg = layer.get_config()
  assert MultiHeadAttention.from_config(cfg).get_config() == cfg
  assert cfg["num_heads"] == 3 and cfg["key_dim"] == 16 and cfg["value_dim"] == 8 and cfg["output_shape"] == 20
  assert MultiHeadAttention(2, 4).get_config()["value_dim"] == 4
  ln = LayerNormalization(epsilon=1e-5, center=False, name="ln")
  cfg = ln.get_config()
  assert LayerNormalization.from_config(cfg).get_config() == cfg
  assert cfg["epsilon"] == 1e-5 and cfg["center"] is False and cfg["scale"] is True and cfg["axis"] == -1


def test_the_head_dim_ceiling_and_the_abi_are_the_headers():
  src = open(os.path.join(ROOT, "include", "tfrs_b200.h")).read()
  assert int(re.search(r"#define TFRS_MHA_MAX_HEAD_DIM (\d+)", src).group(1)) == ops.MHA_MAX_HEAD_DIM == 128
  for name in ("tfrs_mha_fwd_f32", "tfrs_mha_bwd_workspace_bytes", "tfrs_mha_bwd_f32", "tfrs_layer_norm_fwd_f32",
               "tfrs_layer_norm_bwd_workspace_bytes", "tfrs_layer_norm_bwd_f32"):
    assert re.search(name + r"\s*\(", src), name


def test_cpu_tensors_raise():
  x = torch.zeros((2, 3, 4))
  with pytest.raises(RuntimeError, match="CUDA"):
    ops.layer_norm(x)
  with pytest.raises(RuntimeError, match="CUDA"):
    ops.attention_core(x, x, x, 2)
