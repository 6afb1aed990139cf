"""CPU tests of the GRU layer's rule: the float64 oracle (tests/gru_oracle.py) against torch.nn.GRU in float64 and against
finite differences, masking as step removal, the orthogonal initializer, constructor validation, the config round trip
and the ABI declaration of K19."""
import os
import re

import numpy as np
import pytest
import torch

import gru_oracle as go
from recommenders_b200 import ops
from recommenders_b200.layers import GRU
from recommenders_b200.layers.feature_interaction.dcn import _init

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _weights(rng, D, u, bias=True):
  W = rng.uniform(-0.5, 0.5, size=(D, 3 * u))
  U = rng.normal(size=(u, 3 * u)) * 0.6 / np.sqrt(u)
  b = rng.normal(size=(2, 3 * u)) * 0.3 if bias else None
  return W, U, b


def _keras_to_torch(a, u):
  """Keras columns (z, r, h) -> torch.nn.GRU rows (r, z, n)."""
  a = np.asarray(a)
  return np.concatenate([a[..., u:2 * u], a[..., :u], a[..., 2 * u:]], -1).T


@pytest.mark.parametrize("bias", [True, False])
@pytest.mark.parametrize("with_h0", [True, False])
@pytest.mark.parametrize("B,T,D,u", [(3, 5, 4, 6), (1, 1, 1, 1), (4, 7, 9, 3)])
def test_oracle_matches_torch_gru_forward_and_gradients(bias, with_h0, B, T, D, u):
  rng = np.random.RandomState(B * 100 + T * 10 + u)
  x = rng.normal(size=(B, T, D))
  W, U, b = _weights(rng, D, u, bias)
  h0 = rng.normal(size=(B, u)) * 0.5 if with_h0 else None
  g_seq, g_last = rng.normal(size=(B, T, u)), rng.normal(size=(B, u))

  net = torch.nn.GRU(D, u, bias=bias, batch_first=True).double()
  with torch.no_grad():
    net.weight_ih_l0.copy_(torch.from_numpy(_keras_to_torch(W, u)))
    net.weight_hh_l0.copy_(torch.from_numpy(_keras_to_torch(U, u)))
    if bias:
      net.bias_ih_l0.copy_(torch.from_numpy(_keras_to_torch(b[0], u)))
      net.bias_hh_l0.copy_(torch.from_numpy(_keras_to_torch(b[1], u)))
  xt = torch.from_numpy(x).requires_grad_()
  ht = torch.from_numpy(h0 if with_h0 else np.zeros((B, u)))[None].requires_grad_()
  seq_t, hT_t = net(xt, ht)
  (seq_t * torch.from_numpy(g_seq)).sum().add((hT_t[0] * torch.from_numpy(g_last)).sum()).backward()

  seq, hT, _ = go.forward(x, W, U, b, h0)
  np.testing.assert_allclose(seq, seq_t.detach().numpy(), rtol=1e-12, atol=1e-13)
  np.testing.assert_allclose(hT, hT_t[0].detach().numpy(), rtol=1e-12, atol=1e-13)
  g = go.backward(x, W, U, b, h0, None, g_seq, g_last)
  close = lambda a, e: np.testing.assert_allclose(a, e, rtol=1e-10, atol=1e-12)
  close(g["dx"], xt.grad.numpy())
  close(_keras_to_torch(g["dW"], u), net.weight_ih_l0.grad.numpy())
  close(_keras_to_torch(g["dU"], u), net.weight_hh_l0.grad.numpy())
  close(g["dh0"], ht.grad[0].numpy())
  if bias:
    close(_keras_to_torch(g["dbias"][0], u), net.bias_ih_l0.grad.numpy())
    close(_keras_to_torch(g["dbias"][1], u), net.bias_hh_l0.grad.numpy())


def test_oracle_gradients_match_central_differences_with_a_mask():
  rng = np.random.RandomState(7)
  B, T, D, u = 2, 4, 3, 2
  x = rng.normal(size=(B, T, D))
  W, U, b = _weights(rng, D, u)
  h0 = rng.normal(size=(B, u)) * 0.5
  mask = np.array([[1, 0, 1, 1], [0, 1, 1, 0]], bool)
  g_seq, g_last = rng.normal(size=(B, T, u)), rng.normal(size=(B, u))

  def loss(x, W, U, b, h0):
    seq, hT, _ = go.forward(x, W, U, b, h0, mask)
    return float((seq * g_seq).sum() + (hT * g_last).sum())

  g = go.backward(x, W, U, b, h0, mask, g_seq, g_last)
  args = {"dx": x, "dW": W, "dU": U, "dbias": b, "dh0": h0}
  eps = 1e-6
  for name, a in args.items():
    num = np.zeros_like(a)
    for idx in np.ndindex(a.shape):
      keep = a[idx]
      a[idx] = keep + eps; lp = loss(*args.values())
      a[idx] = keep - eps; lm = loss(*args.values())
      a[idx] = keep
      num[idx] = (lp - lm) / (2 * eps)
    np.testing.assert_allclose(g[name], num, rtol=1e-6, atol=1e-8, err_msg=name)
  # the projection's gradient is zero at the masked steps
  assert not g["dgx"][~mask].any()


def test_masked_steps_are_the_same_as_removed_steps():
  rng = np.random.RandomState(3)
  B, T, D, u = 5, 9, 4, 6
  x = rng.normal(size=(B, T, D))
  W, U, b = _weights(rng, D, u)
  h0 = rng.normal(size=(B, u))
  mask = rng.rand(B, T) < 0.6
  mask[3] = False                                  # an all-masked row returns h0
  _, hT, _ = go.forward(x, W, U, b, h0, mask)
  for i in range(B):
    kept = x[i:i + 1, mask[i]]
    exp = h0[i] if kept.shape[1] == 0 else go.forward(kept, W, U, b, h0[i:i + 1])[1][0]
    np.testing.assert_allclose(hT[i], exp, rtol=0, atol=1e-15)
  np.testing.assert_array_equal(hT[3], h0[3])


@pytest.mark.parametrize("shape", [(32, 96), (7, 21), (5, 5), (12, 4), (2, 3, 4)])
def test_orthogonal_initializer(shape):
  torch.manual_seed(0)
  q = _init("orthogonal", shape, "cpu").double().reshape(-1, shape[-1])
  rows, cols = q.shape
  eye = q @ q.T if rows <= cols else q.T @ q
  np.testing.assert_allclose(eye.numpy(), np.eye(min(rows, cols)), atol=1e-6)
  assert _init("orthogonal", shape, "cpu").dtype == torch.float32


def test_orthogonal_initializer_is_seeded():
  torch.manual_seed(5); a = _init("orthogonal", (8, 24), "cpu")
  torch.manual_seed(5); b = _init("orthogonal", (8, 24), "cpu")
  assert torch.equal(a, b)


@pytest.mark.parametrize("kwargs,arg", [
    ({"activation": "relu"}, "activation"), ({"recurrent_activation": "hard_sigmoid"}, "recurrent_activation"),
    ({"reset_after": False}, "reset_after"), ({"dropout": 0.1}, "dropout"),
    ({"recurrent_dropout": 0.2}, "recurrent_dropout"), ({"go_backwards": True}, "go_backwards"),
    ({"stateful": True}, "stateful"), ({"time_major": True}, "time_major")])
def test_unsupported_arguments_raise_naming_the_argument(kwargs, arg):
  with pytest.raises(NotImplementedError, match=arg):
    GRU(8, **kwargs)


def test_units_are_validated_against_the_ceiling():
  GRU(ops.GRU_MAX_UNITS)
  with pytest.raises(ValueError, match=str(ops.GRU_MAX_UNITS)):
    GRU(ops.GRU_MAX_UNITS + 1)
  for bad in (0, -3, 2.5, True):
    with pytest.raises(ValueError):
      GRU(bad)


def test_the_ceiling_is_the_headers():
  src = open(os.path.join(ROOT, "include", "tfrs_b200.h")).read()
  assert int(re.search(r"#define TFRS_GRU_MAX_UNITS (\d+)", src).group(1)) == ops.GRU_MAX_UNITS >= 1024
  for name in ("tfrs_gru_fwd_f32", "tfrs_gru_bwd_workspace_bytes", "tfrs_gru_bwd_f32"):
    assert re.search(name + r"\s*\(", src), name


def test_get_config_round_trip():
  layer = GRU(32, return_sequences=True, return_state=True, use_bias=False, unroll=True, name="q",
              kernel_initializer="truncated_normal")
  cfg = layer.get_config()
  again = GRU.from_config(cfg)
  assert again.get_config() == cfg
  assert cfg["units"] == 32 and cfg["reset_after"] is True and cfg["recurrent_initializer"] == "orthogonal"
  assert cfg["return_sequences"] and cfg["return_state"] and not cfg["use_bias"] and cfg["unroll"]


def test_get_config_round_trip_keeps_a_callable_initializer():
  init = lambda shape, device: torch.full(shape, 0.25, device=device)
  layer = GRU(4, kernel_initializer=init)
  again = GRU.from_config(layer.get_config())
  assert again.get_config()["kernel_initializer"] is init
  again.build((2, 3, 5), device="cpu")
  assert torch.equal(again.kernel.detach(), torch.full((5, 12), 0.25))


def test_cpu_tensors_raise():
  x = torch.zeros((2, 3, 4))
  with pytest.raises(RuntimeError, match="CUDA"):
    ops.gru(x, torch.zeros((4, 6)), torch.zeros((2, 6)))
  with pytest.raises(RuntimeError, match="CUDA"):
    GRU(2)(x, mask=None)
