"""K27 on the CPU: the float64 oracle (tests/conv1d_oracle.py) against torch's conv1d in float64 at every padding, stride,
dilation and kernel size, Keras's output lengths, and `layers.Conv1D`'s argument errors, mask refusal and config."""
import itertools

import numpy as np
import pytest
import torch

import conv1d_oracle as co
import recommenders_b200 as tfrs
from recommenders_b200 import ops


def _torch_conv(x, W, b, s, d, padding):
  """torch.nn.functional.conv1d in float64 on x padded explicitly by the Keras mode's (left, right) pads."""
  T_out, pl, pr = co.geometry(x.shape[1], W.shape[0], s, d, padding)
  xp = torch.nn.functional.pad(x.permute(0, 2, 1), (pl, pr))
  y = torch.nn.functional.conv1d(xp, W.permute(2, 1, 0), b, stride=s, dilation=d).permute(0, 2, 1)
  assert y.shape[1] == T_out
  return y


CASES = [(p, s, d, k) for p, s, d, k in itertools.product(co.PADDINGS, (1, 2, 3), (1, 2, 4), (1, 2, 3, 5))]


@pytest.mark.parametrize("padding,s,d,k", CASES)
def test_oracle_matches_torch_conv1d_forward_and_backward(padding, s, d, k):
  rng = np.random.RandomState(s * 100 + d * 10 + k)
  for T in sorted({1, 2, 7, d * (k - 1) + 1, d * (k - 1) + 2, 13}):
    if co.geometry(T, k, s, d, padding) is None:
      continue
    B, C, F = 3, 4, 5
    x = rng.normal(size=(B, T, C)); W = rng.normal(size=(k, C, F)); b = rng.normal(size=F)
    xt, Wt, bt = (torch.tensor(a, dtype=torch.float64, requires_grad=True) for a in (x, W, b))
    y = _torch_conv(xt, Wt, bt, s, d, padding)
    z, _, _ = co.forward(x, W, b, s, d, padding)
    np.testing.assert_allclose(z, y.detach().numpy(), rtol=1e-12, atol=1e-12)
    g = rng.normal(size=z.shape)
    (y * torch.from_numpy(g)).sum().backward()
    dx, dW, db = co.backward(x, W, g, s, d, padding)
    for got, exp in ((dx, xt.grad), (dW, Wt.grad), (db, bt.grad)):
      np.testing.assert_allclose(got, exp.numpy(), rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("s", [1, 2, 3])
@pytest.mark.parametrize("d", [1, 2, 4])
@pytest.mark.parametrize("k", [1, 2, 3, 5])
def test_output_lengths_follow_keras(s, d, k):
  span = d * (k - 1) + 1
  for T in range(1, 40):
    for padding in co.PADDINGS:
      exp = co.geometry(T, k, s, d, padding)
      if exp is None:
        with pytest.raises(ValueError, match="zero or negative"):
          ops.conv1d_geometry(T, k, s, padding, d)
        continue
      T_out, p = ops.conv1d_geometry(T, k, s, padding, d)
      assert (T_out, p) == exp[:2]
      if padding == "valid":
        assert T_out == (T - d * (k - 1) - 1) // s + 1
      else:
        assert T_out == -(-T // s)
      if padding == "causal":
        assert p == d * (k - 1)
      if padding == "same":   # the extra pad column goes on the right
        assert exp[2] - exp[1] in (0, 1)
  # the valid minimum is one window; one step fewer raises
  assert ops.conv1d_geometry(span, k, s, "valid", d) == (1, 0)
  if span > 1:
    with pytest.raises(ValueError):
      ops.conv1d_geometry(span - 1, k, s, "valid", d)


def test_keras_argument_errors():
  C = tfrs.layers.Conv1D
  with pytest.raises(ValueError, match="filters"):
    C(0, 3)
  with pytest.raises(ValueError, match="filters"):
    C(-2, 3)
  with pytest.raises(ValueError, match="kernel_size"):
    C(4, 0)
  with pytest.raises(ValueError, match="kernel_size"):
    C(4, (3, 3))
  with pytest.raises(ValueError, match="dilation_rate"):
    C(4, 3, dilation_rate=0)
  with pytest.raises(ValueError, match="strides"):
    C(4, 3, strides=-1)
  with pytest.raises(ValueError, match="strides"):
    C(4, 3, strides=0)
  with pytest.raises(ValueError, match="dilation_rate > 1"):
    C(4, 3, strides=2, dilation_rate=2)
  with pytest.raises(ValueError, match="padding"):
    C(4, 3, padding="full")
  with pytest.raises(ValueError, match="data_format"):
    C(4, 3, data_format="nwc")
  with pytest.raises(ValueError, match="Unknown activation"):
    C(4, 3, activation="softplusx")
  with pytest.raises(ValueError, match="divisible"):
    C(4, 3, groups=3)
  assert C(4, 3, padding="CAUSAL").padding == "causal"
  assert C(4.0, [3], strides=(2,)).get_config()["strides"] == (2,)


@pytest.mark.parametrize("kw", [{"groups": 2}, {"data_format": "channels_first"}, {"kernel_regularizer": "l2"},
                                {"bias_regularizer": "l2"}, {"activity_regularizer": "l2"}, {"kernel_constraint": "max_norm"},
                                {"bias_constraint": "max_norm"}])
def test_unsupported_arguments_raise_naming_the_argument(kw):
  with pytest.raises(NotImplementedError, match=next(iter(kw))):
    tfrs.layers.Conv1D(4, 3, **kw)


def test_inputs_of_other_ranks_and_masks_raise():
  layer = tfrs.layers.Conv1D(4, 3, name="title_cnn")
  for shape in ((5, 3), (2, 5, 3, 1)):
    with pytest.raises(NotImplementedError, match="rank"):
      layer(torch.zeros(shape))
  with pytest.raises(TypeError, match="Layer title_cnn does not support masking, but was passed an input_mask"):
    layer(torch.zeros((2, 5, 3)), mask=torch.ones((2, 5), dtype=torch.bool))
  with pytest.raises(TypeError, match="does not support masking"):
    layer(torch.zeros((2, 5, 3)), mask=np.ones((2, 5), bool))
  assert not layer.built
  assert layer.compute_mask(torch.zeros((2, 5, 3))) is None


def test_config_round_trips():
  layer = tfrs.layers.Conv1D(16, 5, strides=1, padding="causal", dilation_rate=4, activation="gelu", use_bias=False,
                             bias_initializer="ones", name="nextitnet_block")
  cfg = layer.get_config()
  again = tfrs.layers.Conv1D.from_config(cfg)
  assert again.get_config() == cfg
  assert cfg["kernel_size"] == (5,) and cfg["dilation_rate"] == (4,) and cfg["activation"] == "gelu"
  assert not cfg["use_bias"] and cfg["name"] == "nextitnet_block"
  assert tfrs.layers.Conv1D.from_config(tfrs.layers.Conv1D(3, 2, activation=torch.tanh).get_config()).get_config()[
      "activation"] == "tanh"
