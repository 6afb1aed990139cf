"""CPU tests of the LSTM layer's rule: the float64 oracle (tests/lstm_oracle.py) against torch.nn.LSTM in float64 and
against finite differences, masking as step removal, constructor validation, `unit_forget_bias`, the config round trip
and the ABI declaration of K20."""
import os
import re

import numpy as np
import pytest
import torch

import lstm_oracle as lo
from recommenders_b200 import ops
from recommenders_b200.layers import LSTM

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _weights(rng, D, u, bias=True):
  W = rng.uniform(-0.5, 0.5, size=(D, 4 * u))
  U = rng.normal(size=(u, 4 * u)) * 0.6 / np.sqrt(u)
  b = rng.normal(size=4 * u) * 0.3 if bias else None
  return W, U, b


@pytest.mark.parametrize("bias", [True, False])
@pytest.mark.parametrize("with_state", [True, False])
@pytest.mark.parametrize("B,T,D,u", [(3, 5, 4, 6), (1, 1, 1, 1), (4, 7, 9, 3)])
def test_oracle_matches_torch_lstm_forward_and_gradients(bias, with_state, B, T, D, u):
  rng = np.random.RandomState(B * 100 + T * 10 + u)
  x = rng.normal(size=(B, T, D))
  W, U, b = _weights(rng, D, u, bias)
  h0 = rng.normal(size=(B, u)) * 0.5 if with_state else None
  c0 = rng.normal(size=(B, u)) if with_state else None
  g_seq, g_h, g_c = rng.normal(size=(B, T, u)), rng.normal(size=(B, u)), rng.normal(size=(B, u))

  # Keras's (i, f, c, o) columns are torch's (i, f, g, o) rows; Keras's one bias is b_ih with b_hh = 0
  net = torch.nn.LSTM(D, u, bias=bias, batch_first=True).double()
  with torch.no_grad():
    net.weight_ih_l0.copy_(torch.from_numpy(W.T))
    net.weight_hh_l0.copy_(torch.from_numpy(U.T))
    if bias:
      net.bias_ih_l0.copy_(torch.from_numpy(b))
      net.bias_hh_l0.zero_()
  xt = torch.from_numpy(x).requires_grad_()
  ht = torch.from_numpy(h0 if with_state else np.zeros((B, u)))[None].requires_grad_()
  ct = torch.from_numpy(c0 if with_state else np.zeros((B, u)))[None].requires_grad_()
  seq_t, (hT_t, cT_t) = net(xt, (ht, ct))
  loss = (seq_t * torch.from_numpy(g_seq)).sum() + (hT_t[0] * torch.from_numpy(g_h)).sum()
  (loss + (cT_t[0] * torch.from_numpy(g_c)).sum()).backward()

  seq, hT, cT, _ = lo.forward(x, W, U, b, h0, c0)
  for got, exp in ((seq, seq_t), (hT, hT_t[0]), (cT, cT_t[0])):
    np.testing.assert_allclose(got, exp.detach().numpy(), rtol=1e-12, atol=1e-13)
  g = lo.backward(x, W, U, b, h0, c0, None, g_seq, g_h, g_c)
  close = lambda a, e: np.testing.assert_allclose(a, e, rtol=1e-10, atol=1e-12)
  close(g["dx"], xt.grad.numpy())
  close(g["dW"].T, net.weight_ih_l0.grad.numpy())
  close(g["dU"].T, net.weight_hh_l0.grad.numpy())
  close(g["dh0"], ht.grad[0].numpy())
  close(g["dc0"], ct.grad[0].numpy())
  if bias:
    close(g["dbias"], net.bias_ih_l0.grad.numpy())


def test_oracle_gradients_match_central_differences_with_a_mask():
  rng = np.random.RandomState(7)
  B, T, D, u = 2, 4, 3, 2
  x = rng.normal(size=(B, T, D))
  W, U, b = _weights(rng, D, u)
  h0, c0 = rng.normal(size=(B, u)) * 0.5, rng.normal(size=(B, u))
  mask = np.array([[1, 0, 1, 1], [0, 1, 1, 0]], bool)
  g_seq, g_h, g_c = rng.normal(size=(B, T, u)), rng.normal(size=(B, u)), rng.normal(size=(B, u))

  def loss(x, W, U, b, h0, c0):
    seq, hT, cT, _ = lo.forward(x, W, U, b, h0, c0, mask)
    return float((seq * g_seq).sum() + (hT * g_h).sum() + (cT * g_c).sum())

  g = lo.backward(x, W, U, b, h0, c0, mask, g_seq, g_h, g_c)
  args = {"dx": x, "dW": W, "dU": U, "dbias": b, "dh0": h0, "dc0": c0}
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
  assert not g["dz"][~mask].any()


def test_masked_steps_are_the_same_as_removed_steps():
  rng = np.random.RandomState(3)
  B, T, D, u = 5, 9, 4, 6
  x = rng.normal(size=(B, T, D))
  W, U, b = _weights(rng, D, u)
  h0, c0 = rng.normal(size=(B, u)), rng.normal(size=(B, u))
  mask = rng.rand(B, T) < 0.6
  mask[3] = False                                  # an all-masked row returns (h0, c0)
  _, hT, cT, _ = lo.forward(x, W, U, b, h0, c0, mask)
  for i in range(B):
    kept = x[i:i + 1, mask[i]]
    if kept.shape[1] == 0:
      eh, ec = h0[i], c0[i]
    else:
      _, eh, ec, _ = lo.forward(kept, W, U, b, h0[i:i + 1], c0[i:i + 1])
      eh, ec = eh[0], ec[0]
    np.testing.assert_allclose(hT[i], eh, rtol=0, atol=1e-15)
    np.testing.assert_allclose(cT[i], ec, rtol=0, atol=1e-15)
  np.testing.assert_array_equal(hT[3], h0[3])
  np.testing.assert_array_equal(cT[3], c0[3])


@pytest.mark.parametrize("kwargs,arg", [
    ({"activation": "relu"}, "activation"), ({"recurrent_activation": "hard_sigmoid"}, "recurrent_activation"),
    ({"dropout": 0.1}, "dropout"), ({"recurrent_dropout": 0.2}, "recurrent_dropout"),
    ({"go_backwards": True}, "go_backwards"), ({"stateful": True}, "stateful"), ({"time_major": True}, "time_major")])
def test_unsupported_arguments_raise_naming_the_argument(kwargs, arg):
  with pytest.raises(NotImplementedError, match=arg):
    LSTM(8, **kwargs)


def test_implementation_and_unroll_are_accepted():
  for kw in ({"implementation": 1}, {"implementation": 2}, {"unroll": True}):
    LSTM(8, **kw)


def test_units_are_validated_against_the_ceiling():
  LSTM(ops.LSTM_MAX_UNITS)
  with pytest.raises(ValueError, match=str(ops.LSTM_MAX_UNITS)):
    LSTM(ops.LSTM_MAX_UNITS + 1)
  for bad in (0, -3, 2.5, True):
    with pytest.raises(ValueError):
      LSTM(bad)


def test_the_ceiling_is_the_headers():
  src = open(os.path.join(ROOT, "include", "tfrs_b200.h")).read()
  assert int(re.search(r"#define TFRS_LSTM_MAX_UNITS (\d+)", src).group(1)) == ops.LSTM_MAX_UNITS >= 1024
  for name in ("tfrs_lstm_fwd_f32", "tfrs_lstm_bwd_workspace_bytes", "tfrs_lstm_bwd_f32"):
    assert re.search(name + r"\s*\(", src), name


@pytest.mark.parametrize("unit_forget_bias", [True, False])
def test_build_shapes_and_unit_forget_bias(unit_forget_bias):
  torch.manual_seed(0)
  u, D = 6, 5
  layer = LSTM(u, unit_forget_bias=unit_forget_bias, bias_initializer="zeros")
  layer.build((2, 3, D), device="cpu")
  assert layer.kernel.shape == (D, 4 * u) and layer.recurrent_kernel.shape == (u, 4 * u) and layer.bias.shape == (4 * u,)
  b = layer.bias.detach()
  assert torch.equal(b[u:2 * u], torch.full((u,), 1.0 if unit_forget_bias else 0.0))
  assert not b[:u].any() and not b[2 * u:].any()
  rk = layer.recurrent_kernel.detach().double()
  np.testing.assert_allclose((rk @ rk.T).numpy(), np.eye(u), atol=1e-6)
  nobias = LSTM(u, use_bias=False)
  nobias.build((2, 3, D), device="cpu")
  assert nobias.bias is None


def test_unit_forget_bias_calls_the_bias_initializer_per_slice():
  shapes = []

  def init(shape, device):
    shapes.append(tuple(shape))
    return torch.full(shape, 0.5, device=device)

  layer = LSTM(3, bias_initializer=init)
  layer.build((1, 1, 2), device="cpu")
  assert shapes == [(3,), (6,)]
  assert torch.equal(layer.bias.detach(), torch.tensor([0.5] * 3 + [1.0] * 3 + [0.5] * 6))


def test_get_config_round_trip():
  layer = LSTM(32, return_sequences=True, return_state=True, use_bias=False, unroll=True, name="q",
               kernel_initializer="truncated_normal", unit_forget_bias=False, implementation=1)
  cfg = layer.get_config()
  again = LSTM.from_config(cfg)
  assert again.get_config() == cfg
  assert cfg["units"] == 32 and cfg["recurrent_initializer"] == "orthogonal" and cfg["unit_forget_bias"] is False
  assert cfg["return_sequences"] and cfg["return_state"] and not cfg["use_bias"] and cfg["unroll"]
  assert LSTM(4).get_config()["unit_forget_bias"] is True


def test_get_config_round_trip_keeps_a_callable_initializer():
  init = lambda shape, device: torch.full(shape, 0.25, device=device)
  layer = LSTM(4, kernel_initializer=init)
  again = LSTM.from_config(layer.get_config())
  assert again.get_config()["kernel_initializer"] is init
  again.build((2, 3, 5), device="cpu")
  assert torch.equal(again.kernel.detach(), torch.full((5, 16), 0.25))


def test_cpu_tensors_raise():
  x = torch.zeros((2, 3, 4))
  with pytest.raises(RuntimeError, match="CUDA"):
    ops.lstm(x, torch.zeros((4, 8)), torch.zeros((2, 8)))
  with pytest.raises(RuntimeError, match="CUDA"):
    LSTM(2)(x, mask=None)
