"""CPU tests of FTRL: the fp32 oracle (tests/ftrl_oracle.py) against the float64 rule and TF's ftrl_test.py known answers,
its sparse rule, and the checks of the public class that run before any kernel."""
import itertools
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import ftrl_oracle as fo  # noqa: E402


def bits(a):
  return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _close(got, want):
  """1e-6 relative; elements that pass near zero (the linear slot is a running sum of signed terms, and a weight next to
  the l1 threshold is near zero) are held to 1e-6 of the tensor's scale."""
  np.testing.assert_allclose(got, want, rtol=1e-6, atol=1e-6 * np.abs(want).max())


_SETTINGS = {"plain": {}, "l1": dict(l1=0.05), "l2": dict(l2=0.5), "shrinkage": dict(l2_shrinkage=0.2),
             "beta": dict(beta=0.7), "all": dict(l1=0.05, l2=0.5, l2_shrinkage=0.2, beta=0.7)}


@pytest.mark.parametrize("lr_power,setting", list(itertools.product((-0.5, 0.0, -1.0, -0.3), sorted(_SETTINGS))))
def test_oracle_tracks_the_float64_rule(lr_power, setting):
  """20 steps of the fp32 rule agree with the float64 rule within 1e-6 relative."""
  kw = dict(_SETTINGS[setting], lr=0.1, lr_power=lr_power)
  rng = np.random.RandomState(0)
  x = rng.uniform(-1, 1, size=(64, 8)).astype(np.float32)
  a = np.full_like(x, 0.1); z = np.zeros_like(x)
  x64, a64, z64 = x.astype(np.float64), a.astype(np.float64), z.astype(np.float64)
  f64 = {k: float(np.float32(v)) for k, v in kw.items()}
  for _ in range(20):
    g = rng.normal(size=x.shape).astype(np.float32)
    x, a, z = fo.ftrl_dense(x, a, z, g, **kw)
    x64, a64, z64 = fo.ftrl_textbook(x64, a64, z64, g, **f64)
    for got, want in ((x, x64), (a, a64), (z, z64)):
      assert got.dtype == np.float32
      _close(got, want)


# TF's ftrl_test.py: lr = 3.0, initial accumulator 0.1, gradients [0.1, 0.2] (var0) and [0.01, 0.02] (var1) every step.
_KNOWN = [
    ({}, [0., 0.], [0., 0.], 3, [-2.60260963, -4.29698515], [-0.28432083, -0.56694895]),
    (dict(l1=0.001), [1., 2.], [4., 3.], 10, [-7.66718769, -10.91273689], [-0.93460727, -1.86147261]),
    (dict(l1=0.001, l2=2.0), [1., 2.], [4., 3.], 10, [-0.24059935, -0.46829352], [-0.02406147, -0.04830509]),
    (dict(l1=0.001, l2=2.0, l2_shrinkage=0.1), [1., 2.], [4., 3.], 10, [-0.22578995, -0.44345796],
     [-0.14378493, -0.13229476]),
]


@pytest.mark.parametrize("kw,start0,start1,steps,want0,want1", _KNOWN)
@pytest.mark.parametrize("rule", ["fp32", "float64"])
def test_tf_known_answers(kw, start0, start1, steps, want0, want1, rule):
  step = fo.ftrl_dense if rule == "fp32" else fo.ftrl_textbook
  for start, grad, want in ((start0, [0.1, 0.2], want0), (start1, [0.01, 0.02], want1)):
    x = np.array(start, np.float32); a = np.full(2, 0.1, np.float32); z = np.zeros(2, np.float32)
    for _ in range(steps):
      x, a, z = step(x, a, z, np.array(grad, np.float32), lr=3.0, **kw)
    np.testing.assert_allclose(np.asarray(x, np.float64), want, rtol=1e-6, atol=1e-6)


@pytest.mark.parametrize("lr_power", [-0.5, -0.3])
def test_l1_sets_exact_positive_zeros(lr_power):
  """Every element with |lin'| <= l1 gets var' == +0 bit for bit, and the others do not."""
  rng = np.random.RandomState(4)
  x = rng.uniform(-1, 1, size=(4096,)).astype(np.float32)
  a = np.full_like(x, 0.1); z = rng.uniform(-1, 1, size=x.shape).astype(np.float32)
  g = rng.normal(size=x.shape).astype(np.float32)
  l1 = 0.5
  x1, _, z1 = fo.ftrl_dense(x, a, z, g, lr=0.1, lr_power=lr_power, l1=l1, l2=0.1)
  inside = np.abs(z1) <= np.float32(l1)
  assert 100 < inside.sum() < x.size - 100
  assert (bits(x1[inside]) == 0).all()
  assert (x1[~inside] != 0).all() and (np.sign(x1[~inside]) == -np.sign(z1[~inside])).all()


def test_lr_power_zero_is_sgd():
  """lr_power = 0 and no regularization, from var = 0: P = 1, so var' = -lin'/(1/lr) = -lr * (sum of the gradients)."""
  rng = np.random.RandomState(5)
  x = np.zeros((256,), np.float32); a = np.full_like(x, 0.1); z = np.zeros_like(x)
  total = np.zeros(x.shape, np.float64)
  for _ in range(5):
    g = rng.normal(size=x.shape).astype(np.float32)
    x, a, z = fo.ftrl_dense(x, a, z, g, lr=0.05, lr_power=0.0)
    total += g
  np.testing.assert_allclose(z, total, rtol=1e-5, atol=1e-6)
  np.testing.assert_allclose(x, -float(np.float32(0.05)) * z.astype(np.float64), rtol=3e-7)


def test_power_modes():
  """sqrt for lr_power = -0.5 (TF's special case); otherwise float64 pow rounded once, so lr_power = 0 gives exactly 1."""
  x = np.array([0.1, 1.0, 2.5, 1e-30, 7e20], np.float32)
  assert np.array_equal(bits(fo.power(x, -0.5)), bits(np.sqrt(x)))
  assert np.array_equal(fo.power(x, 0.0), np.ones_like(x))
  want = (x.astype(np.float64) ** np.float64(np.float32(0.3))).astype(np.float32)
  assert np.array_equal(bits(fo.power(x, -0.3)), bits(want))


def test_sparse_oracle_sums_duplicates_in_order_skips_out_of_range_and_keeps_other_rows():
  rng = np.random.RandomState(2)
  x = rng.uniform(-1, 1, size=(6, 3)).astype(np.float32)
  a = rng.uniform(0.1, 1, size=x.shape).astype(np.float32); z = rng.uniform(-1, 1, size=x.shape).astype(np.float32)
  g = np.array([[0.5, 0.25, 1e-8], [0.125, 1., -3.], [9., 9., 9.], [1e8, -0.5, 3.], [7., 7., 7.], [-1e8, 2., 1.]],
               np.float32)
  ids = np.array([0, 1, -1, 0, 6, 0])
  summed = np.stack([(g[0] + g[3]) + g[5], g[1]])
  assert not np.array_equal(bits(summed[0]), bits(g[0] + (g[3] + g[5])))   # the order matters for these rows
  kw = dict(lr=0.1, l1=0.01, l2=0.1, l2_shrinkage=0.05)
  got = fo.ftrl_sparse(x, a, z, ids, g, **kw)
  want = fo.ftrl_sparse(x, a, z, np.array([0, 1]), summed, **kw)
  dense = fo.ftrl_dense(x[:2], a[:2], z[:2], summed, **kw)
  for p, q, r, was in zip(got, want, dense, (x, a, z)):
    assert np.array_equal(bits(p), bits(q))
    assert np.array_equal(bits(p[:2]), bits(r))
    assert np.array_equal(bits(p[2:]), bits(was[2:]))


def test_ftrl_l2_folds_beta_in_fp32():
  from recommenders_b200 import ops
  for l2, beta, lr in itertools.product((0.0, 2.0, 0.3), (0.0, 0.1, 7.3), (3.0, 0.1, 1e-3, 0.7)):
    got = ops.ftrl_l2(l2, beta, lr)
    assert got == float(fo.l2a(l2, beta, lr))
    assert got == float(np.float32(np.float32(l2) + np.float32(np.float32(beta) / (np.float32(2) * np.float32(lr)))))


def test_ftrl_constructor_config_and_errors():
  from recommenders_b200.optimizers import Ftrl
  opt = Ftrl()
  assert (opt.learning_rate, opt.learning_rate_power, opt.initial_accumulator_value, opt.l1_regularization_strength,
          opt.l2_regularization_strength, opt.name, opt.l2_shrinkage_regularization_strength, opt.beta) == (
              0.001, -0.5, 0.1, 0.0, 0.0, "Ftrl", 0.0, 0.0)
  assert opt.iterations == 0 and opt.variables() == []
  # tf-keras's positional order
  opt = Ftrl(0.3, -0.25, 0.2, 0.01, 0.02, "ftrl2", 0.03, 0.4)
  config = opt.get_config()
  assert config == {"learning_rate": 0.3, "learning_rate_power": -0.25, "initial_accumulator_value": 0.2,
                    "l1_regularization_strength": 0.01, "l2_regularization_strength": 0.02, "name": "ftrl2",
                    "l2_shrinkage_regularization_strength": 0.03, "beta": 0.4}
  restored = Ftrl.from_config(config)
  for attr in config:
    assert getattr(restored, attr) == getattr(opt, attr), attr
  assert restored.get_config() == config
  Ftrl(initial_accumulator_value=0.0, learning_rate_power=0.0)   # the edges are allowed
  for kw, match in ((dict(initial_accumulator_value=-0.1), "initial_accumulator_value"),
                    (dict(learning_rate_power=0.5), "learning_rate_power"),
                    (dict(l1_regularization_strength=-1e-3), "l1_regularization_strength"),
                    (dict(l2_regularization_strength=-1e-3), "l2_regularization_strength"),
                    (dict(l2_shrinkage_regularization_strength=-1e-3), "l2_shrinkage_regularization_strength")):
    with pytest.raises(ValueError, match=match):
      Ftrl(**kw)
