"""CPU tests of the Dropout and BatchNormalization rules: the NumPy Philox4x32-10 against Random123's known answers, the
dropout oracle's mask rules, the float64 batch-norm oracle against float64 torch (F.batch_norm and autograd) and against
central differences on a masked case, the training-phase resolution order, constructor errors, configs and the ABI
declarations of K23 / K24."""
import math
import os
import re

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import regularization_oracle as ro
from recommenders_b200 import _ffi, backend, ops
from recommenders_b200.layers import BatchNormalization, Dropout, SpatialDropout1D

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
U = 0xFFFFFFFF


@pytest.mark.parametrize("ctr,key,expected", [
    ((0, 0, 0, 0), (0, 0), (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
    ((U, U, U, U), (U, U), (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
    ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0),
     (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1)),
])
def test_philox_matches_random123_known_answers(ctr, key, expected):
  assert tuple(int(w) for w in ro.philox4x32_10(ctr, key)) == expected


def test_the_mask_takes_word_j_mod_4_of_counter_j_div_4():
  seed, call = 0x0123456789ABCDEF, (7 << 32) | 3
  keep = ro.dropout_keep((11,), 0.5, seed, call)
  for j in range(11):
    w = ro.philox4x32_10((j // 4, 0, 3, 7), (0x89ABCDEF, 0x01234567))[j % 4]
    assert keep[j] == ((int(w) >> 8) >= ro.threshold(0.5))


def test_threshold_scale_and_dropped_values():
  assert ro.threshold(0.0) == 0 and ro.threshold(2.0**-24) == 1 and ro.threshold(0.5) == 2**23
  assert ro.threshold(0.1) == math.ceil(0.1 * 2**24)
  assert ro.scale_of(0.1) == np.float32(1 / 0.9)
  x = np.array([np.nan, np.inf, -np.inf, -0.0, 1.0] * 200, np.float32)
  y = ro.dropout(x, 0.5, 1, 0)
  keep = ro.dropout_keep(x.shape, 0.5, 1, 0)
  assert np.all(np.signbit(y[~keep]) == False) and np.all(y[~keep] == 0)   # noqa: E712 (+0, never NaN or inf)
  assert np.array_equal(np.isnan(y), np.isnan(x) & keep)
  assert np.array_equal(ro.dropout(x, 0.0, 1, 0), x * np.float32(1.0), equal_nan=True)


def test_broadcast_noise_shapes_repeat_one_mask_value():
  x = np.ones((3, 5, 4), np.float32)
  y = ro.dropout(x, 0.5, 9, 2, noise_shape=(None, 1, None))
  assert np.array_equal(y, np.broadcast_to(y[:, :1], y.shape))
  keep = ro.dropout_keep((3, 1, 4), 0.5, 9, 2)
  assert np.array_equal(y != 0, np.broadcast_to(keep, x.shape))


def test_the_keep_fraction_is_binomial():
  n, rate = 1 << 20, 0.3
  kept = ro.dropout_keep((n,), rate, 1234, 0).sum()
  p = 1 - ro.threshold(rate) / 2**24
  assert abs(kept - n * p) <= 6 * math.sqrt(n * p * (1 - p))


# ---- batch normalization ----------------------------------------------------------------------------------------
def _torch_bn(x, gamma, beta, dy, eps=1e-3):
  xt, gt, bt = (torch.tensor(a, dtype=torch.float64, requires_grad=True) for a in (x, gamma, beta))
  y = F.batch_norm(xt.reshape(-1, x.shape[-1]), None, None, gt, bt, training=True, eps=float(np.float32(eps)))
  y.backward(torch.tensor(dy.reshape(-1, x.shape[-1])))
  return y.detach().numpy().reshape(x.shape), xt.grad.numpy(), gt.grad.numpy(), bt.grad.numpy()


@pytest.mark.parametrize("shape", [(2, 3), (7, 5), (64, 33), (4, 9, 6)])
def test_batch_norm_oracle_matches_torch_in_training(shape):
  rng = np.random.RandomState(sum(shape))
  x, dy = rng.normal(size=shape) * 3 + 2, rng.normal(size=shape)
  gamma, beta = rng.normal(size=shape[-1]), rng.normal(size=shape[-1])
  mm, mv = rng.normal(size=shape[-1]), rng.rand(shape[-1]) + 0.5
  y, nmm, nmv = ro.batch_norm_forward(x, gamma, beta, mm, mv, True, 0.9)
  dx, dg, db = ro.batch_norm_backward(x, gamma, dy, mm, mv, True)
  ty, tdx, tdg, tdb = _torch_bn(x, gamma, beta, dy)
  for a, b in ((y, ty), (dx, tdx), (dg, tdg), (db, tdb)):
    np.testing.assert_allclose(a, b, rtol=1e-10, atol=1e-10)
  # the moving update by its formula on the population variance (torch's running variance is unbiased)
  x2 = x.reshape(-1, shape[-1])
  decay = float(np.float32(1 - 0.9))
  np.testing.assert_allclose(nmm, mm - (mm - x2.mean(0)) * decay, rtol=1e-12)
  np.testing.assert_allclose(nmv, mv - (mv - x2.var(0)) * decay, rtol=1e-12)


def test_batch_norm_oracle_at_inference_matches_torch():
  rng = np.random.RandomState(3)
  x, dy = rng.normal(size=(20, 7)), rng.normal(size=(20, 7))
  gamma, beta, mm, mv = rng.normal(size=7), rng.normal(size=7), rng.normal(size=7), rng.rand(7) + 0.5
  y, nmm, nmv = ro.batch_norm_forward(x, gamma, beta, mm, mv, False)
  assert np.array_equal(nmm, mm) and np.array_equal(nmv, mv)
  xt, gt, bt = (torch.tensor(a, requires_grad=True) for a in (x, gamma, beta))
  ty = F.batch_norm(xt, torch.tensor(mm), torch.tensor(mv), gt, bt, training=False, eps=float(np.float32(1e-3)))
  ty.backward(torch.tensor(dy))
  dx, dg, db = ro.batch_norm_backward(x, gamma, dy, mm, mv, False)
  for a, b in ((y, ty.detach()), (dx, xt.grad), (dg, gt.grad), (db, bt.grad)):
    np.testing.assert_allclose(a, b.numpy(), rtol=1e-10, atol=1e-12)


def test_masked_batch_norm_backward_matches_central_differences():
  rng = np.random.RandomState(5)
  B, T, d = 3, 4, 5
  x, dy = rng.normal(size=(B, T, d)) + 1.5, rng.normal(size=(B, T, d))
  gamma, beta = rng.normal(size=d), rng.normal(size=d)
  mask = rng.rand(B, T) < 0.6
  mask[0, 0], mask[1, 1] = True, False
  mm, mv = np.zeros(d), np.ones(d)
  loss = lambda xx, gg, bb: float((ro.batch_norm_forward(xx, gg, bb, mm, mv, True, mask=mask)[0] * dy).sum())
  dx, dg, db = ro.batch_norm_backward(x, gamma, dy, mm, mv, True, mask=mask)
  h = 1e-6
  for arr, grad in ((x, dx), (gamma, dg), (beta, db)):
    num = np.zeros_like(arr)
    for i in np.ndindex(arr.shape):
      e = np.zeros_like(arr)
      e[i] = h
      args = [x, gamma, beta]
      k = next(j for j, a in enumerate(args) if a is arr)
      plus, minus = list(args), list(args)
      plus[k], minus[k] = arr + e, arr - e
      num[i] = (loss(*plus) - loss(*minus)) / (2 * h)
    np.testing.assert_allclose(grad, num, rtol=1e-5, atol=1e-6)
  # masked rows do not move the moments
  mean, var, n = ro.batch_moments(x, mask)
  np.testing.assert_allclose(mean, x[mask].mean(0)) and np.testing.assert_allclose(var, x[mask].var(0))
  assert n == mask.sum()


def test_an_all_masked_batch_has_mean_0_and_variance_0():
  x = np.random.RandomState(0).normal(size=(6, 3))
  mean, var, n = ro.batch_moments(x, np.zeros(6, bool))
  assert n == 0 and not mean.any() and not var.any()
  dx, _, _ = ro.batch_norm_backward(x, None, np.ones((6, 3)), None, None, True, mask=np.zeros(6, bool))
  np.testing.assert_allclose(dx, np.full((6, 3), 1 / math.sqrt(float(np.float32(1e-3)))))


# ---- the training phase -------------------------------------------------------------------------------------------
def test_training_resolves_argument_then_innermost_scope_then_false():
  assert backend.resolve_training() is False and backend.learning_phase() is None
  assert backend.resolve_training(True) is True
  with backend.learning_phase_scope(True):
    assert backend.resolve_training() is True and backend.resolve_training(False) is False
    with backend.learning_phase_scope(False):
      assert backend.resolve_training() is False and backend.resolve_training(True) is True
    assert backend.resolve_training() is True
  assert backend.resolve_training() is False


def test_train_and_test_steps_open_their_phase():
  import recommenders_b200 as tfrs
  seen = []

  class M(tfrs.Model):
    def __init__(self):
      super().__init__()
      self.w = torch.nn.Parameter(torch.zeros(()))

    def compute_loss(self, inputs, training=False):
      seen.append(backend.resolve_training())
      return self.w * 0

  class Opt:
    def zero_grad(self):
      pass

    def apply_gradients(self):
      pass

  m = M()
  m.optimizer = Opt()
  m.train_step(None)
  m.test_step(None)
  assert seen == [True, False] and backend.learning_phase() is None


def test_dropout_at_inference_returns_the_input_without_a_device():
  x = torch.ones(3)
  layer = Dropout(0.5, seed=1)
  assert layer(x) is x and layer(x, training=False) is x
  with backend.learning_phase_scope(False):
    assert layer(x) is x
  with backend.learning_phase_scope(True):
    assert Dropout(0.0)(x) is x
    with pytest.raises(RuntimeError, match="CUDA"):
      layer(x)


# ---- constructors, configs, ABI -------------------------------------------------------------------------------------
@pytest.mark.parametrize("rate", [-0.1, 1.0, 1.5])
def test_dropout_rate_errors(rate):
  with pytest.raises(ValueError, match="rate"):
    Dropout(rate)
  with pytest.raises(ValueError, match="rate"):
    SpatialDropout1D(rate)


def test_dropout_configs_round_trip_and_seeds():
  layer = Dropout(0.2, noise_shape=(None, 1, None), seed=7)
  again = Dropout.from_config(layer.get_config())
  assert again.get_config() == layer.get_config() == {"rate": 0.2, "noise_shape": (None, 1, None), "seed": 7, "name": None}
  assert again._key == layer._key == 7
  s = SpatialDropout1D(0.3, seed=2)
  assert SpatialDropout1D.from_config(s.get_config()).get_config() == s.get_config()
  torch.manual_seed(11)
  k1 = Dropout(0.1)._key
  torch.manual_seed(11)
  assert Dropout(0.1)._key == k1 and Dropout(0.1)._key != k1
  assert Dropout(0.1, seed=-1)._key == 2**64 - 1


def test_dropout_noise_shape_checks():
  assert ops.dropout_noise_shape((4, 5, 6), (None, 1, None)) == (4, 1, 6)
  with pytest.raises(ValueError, match="noise_shape"):
    ops.dropout_noise_shape((4, 5, 6), (4, 2, 6))
  with pytest.raises(ValueError, match="noise_shape"):
    ops.dropout_noise_shape((4, 5), (4, 5, 1))
  with pytest.raises(ValueError, match="noise_shape"):
    ops.dropout_noise_shape((4, 5), (4, 5, None))


@pytest.mark.parametrize("arg,value", [("renorm", True), ("virtual_batch_size", 8), ("adjustment", lambda s: s),
                                       ("synchronized", True), ("beta_regularizer", "l2"), ("gamma_regularizer", "l2"),
                                       ("beta_constraint", "non_neg"), ("gamma_constraint", "non_neg"),
                                       ("renorm_clipping", {}), ("trainable", False)])
def test_batch_norm_unsupported_arguments(arg, value):
  with pytest.raises(NotImplementedError, match=arg):
    BatchNormalization(**{arg: value})


def test_batch_norm_axis_and_config():
  with pytest.raises(NotImplementedError, match="axis"):
    BatchNormalization(axis=[1, 2])
  with pytest.raises(NotImplementedError, match="axis"):
    BatchNormalization(axis=1)._check_axis(3)
  layer = BatchNormalization(momentum=0.9, epsilon=1e-5, center=False)
  again = BatchNormalization.from_config(layer.get_config())
  assert again.get_config() == layer.get_config()
  assert layer.get_config()["momentum"] == 0.9 and layer.get_config()["center"] is False


def test_abi_declarations():
  src = open(os.path.join(ROOT, "include", "tfrs_b200.h")).read()
  assert int(re.search(r"#define TFRS_DROPOUT_MAX_RANK (\d+)", src).group(1)) == ops.DROPOUT_MAX_RANK == 4
  for name in ("tfrs_dropout_f32", "tfrs_batch_norm_fwd_workspace_bytes", "tfrs_batch_norm_fwd_f32",
               "tfrs_batch_norm_bwd_workspace_bytes", "tfrs_batch_norm_bwd_f32"):
    assert re.search(name + r"\s*\(", src), name
    assert name in _ffi.EXPORTS
