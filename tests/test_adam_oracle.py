"""CPU tests of Adam: the fp32 oracle (tests/adam_oracle.py) against TF's textbook float64 update (adam_update_numpy),
its sparse rules, and the checks of the public class that run before any kernel."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import adam_oracle as ao  # noqa: E402


def bits(a):
  return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _close(got, want):
  """1e-6 relative; elements that pass near zero (a variable crossing it, m as a running sum of signed gradients) are
  held to 1e-6 of the tensor's scale."""
  np.testing.assert_allclose(got, want, rtol=1e-6, atol=1e-6 * np.abs(want).max())


@pytest.mark.parametrize("beta_1,beta_2,epsilon,lr", [(0.9, 0.999, 1e-7, 0.001), (0.5, 0.9, 1e-3, 0.1),
                                                      (0.95, 0.99, 1e-8, 0.01)])
def test_dense_oracle_tracks_the_textbook_update(beta_1, beta_2, epsilon, lr):
  """20 steps of the fp32 dense rule agree with the float64 textbook form within 1e-6 relative."""
  rng = np.random.RandomState(0)
  x = rng.uniform(-1, 1, size=(64, 8)).astype(np.float32)
  m = np.zeros_like(x); v = np.zeros_like(x)
  x64, m64, v64 = x.astype(np.float64), m.astype(np.float64), v.astype(np.float64)
  for t in range(1, 21):
    g = rng.normal(size=x.shape).astype(np.float32)
    x, m, v = ao.adam_dense(x, m, v, g, lr, t, beta_1, beta_2, epsilon)
    b1, b2 = float(np.float32(beta_1)), float(np.float32(beta_2))
    x64, m64, v64 = ao.adam_textbook(x64, m64, v64, g, float(np.float32(lr)), t, b1, b2, float(np.float32(epsilon)))
    for got, want in ((x, x64), (m, m64), (v, v64)):
      _close(got, want)


@pytest.mark.parametrize("lazy", [False, True])
def test_sparse_oracle_tracks_the_textbook_update(lazy):
  """Every id touched on every step: both sparse rules are the dense rule up to rounding (20 steps, 1e-6 relative)."""
  rng = np.random.RandomState(1)
  x = rng.uniform(-1, 1, size=(16, 4)).astype(np.float32)
  m = np.zeros_like(x); v = np.zeros_like(x)
  x64, m64, v64 = x.astype(np.float64), m.astype(np.float64), v.astype(np.float64)
  for t in range(1, 21):
    g = rng.normal(size=x.shape).astype(np.float32)
    x, m, v = ao.adam_sparse(x, m, v, np.arange(16), g, 0.01, t, lazy=lazy)
    x64, m64, v64 = ao.adam_textbook(x64, m64, v64, g, float(np.float32(0.01)), t, float(np.float32(0.9)),
                                     float(np.float32(0.999)), float(np.float32(1e-7)))
    for got, want in ((x, x64), (m, m64), (v, v64)):
      _close(got, want)


def test_alpha_is_rounded_once_from_fp32_hyperparameters():
  a = ao.alpha(0.001, 0.9, 0.999, 1)
  b1, b2, lr = (float(np.float32(s)) for s in (0.9, 0.999, 0.001))
  assert a == np.float32(lr * np.sqrt(1 - b2) / (1 - b1)) and a.dtype == np.float32
  from recommenders_b200 import ops
  for t in (1, 2, 7, 1000):
    for lr, b1, b2 in ((0.001, 0.9, 0.999), (0.3, 0.5, 0.75), (1e-5, 0.99, 0.9999)):
      assert ops.adam_alpha(lr, b1, b2, t) == float(ao.alpha(lr, b1, b2, t))


@pytest.mark.parametrize("lazy", [False, True])
def test_sparse_oracle_sums_duplicates_in_order_and_skips_out_of_range(lazy):
  rng = np.random.RandomState(2)
  x = rng.uniform(-1, 1, size=(5, 3)).astype(np.float32)
  m = rng.uniform(-0.1, 0.1, size=x.shape).astype(np.float32); v = rng.uniform(0, 0.1, size=x.shape).astype(np.float32)
  g = np.array([[0.5, 0.25, 1e-8], [0.125, 1., -3.], [9., 9., 9.], [1e8, -0.5, 3.], [7., 7., 7.], [-1e8, 2., 1.]],
               np.float32)
  ids = np.array([0, 1, -1, 0, 5, 0])
  summed = np.stack([(g[0] + g[3]) + g[5], g[1]])
  assert not np.array_equal(bits(summed[0]), bits(g[0] + (g[3] + g[5])))   # the order matters for these rows
  a = ao.adam_sparse(x, m, v, ids, g, 0.01, 3, lazy=lazy)
  b = ao.adam_sparse(x, m, v, np.array([0, 1]), summed, 0.01, 3, lazy=lazy)
  for p, q in zip(a, b):
    assert np.array_equal(bits(p), bits(q))


def test_lazy_leaves_untouched_rows_bit_identical():
  rng = np.random.RandomState(3)
  x = rng.uniform(-1, 1, size=(50, 8)).astype(np.float32)
  m = rng.uniform(-0.1, 0.1, size=x.shape).astype(np.float32); v = rng.uniform(0, 0.1, size=x.shape).astype(np.float32)
  ids = np.array([3, 7, 7, 49, 50, -2])
  g = rng.normal(size=(ids.size, 8)).astype(np.float32)
  lx, lm, lv = ao.adam_sparse(x, m, v, ids, g, 0.01, 5, lazy=True)
  nx, nm, nv = ao.adam_sparse(x, m, v, ids, g, 0.01, 5, lazy=False)
  other = np.setdiff1d(np.arange(50), [3, 7, 49])
  for got, was in ((lx, x), (lm, m), (lv, v)):
    assert np.array_equal(bits(got[other]), bits(was[other]))
  touched = [3, 7, 49]
  for p, q in ((lx, nx), (lm, nm), (lv, nv)):
    assert np.array_equal(bits(p[touched]), bits(q[touched]))
  # not lazy: every untouched row decays and moves
  assert (nm[other] != m[other]).all() and (nx[other] != x[other]).any()


def test_adam_constructor_config_and_amsgrad():
  from recommenders_b200.optimizers import Adam
  opt = Adam()
  assert (opt.learning_rate, opt.beta_1, opt.beta_2, opt.epsilon, opt.amsgrad, opt.lazy_embeddings, opt.name) == (
      0.001, 0.9, 0.999, 1e-7, False, False, "Adam")
  assert opt.iterations == 0 and opt.variables() == []
  opt = Adam(learning_rate=0.01, beta_1=0.8, beta_2=0.99, epsilon=1e-5, lazy_embeddings=True, name="adam2")
  config = opt.get_config()
  assert set(config) == {"learning_rate", "beta_1", "beta_2", "epsilon", "amsgrad", "lazy_embeddings", "name"}
  restored = Adam.from_config(config)
  for attr in config:
    assert getattr(restored, attr) == getattr(opt, attr), attr
  with pytest.raises(NotImplementedError, match="amsgrad"):
    Adam(amsgrad=True)
