"""CPU tests of the ClippyAdagrad / CompositeOptimizer additions: the reference's known answers
(experimental/optimizers/clippy_adagrad_test.py, composite_optimizer_test.py) restated against the oracle, and the
checks of the public classes that run before any kernel."""
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import clippy_oracle as co  # noqa: E402

F32_TOL = dict(rtol=1e-6, atol=1e-6)   # assertAllCloseAccordingToType for float32


def _close(actual, expected, **tol):
  np.testing.assert_allclose(np.asarray(actual, np.float64), np.asarray(expected, np.float64), **(tol or F32_TOL))


# ---- ClipByReferenceTest (clippy_adagrad_test.py:21-160), float64 -------------------------------------------------------
@pytest.mark.parametrize("tensor,references,relative_factors,absolute_factor,expected", [
    (2., [4.], [0.1], 0.02, (0.42, 0.21)),
    (2., [-4.], [0.1], 0.02, (0.42, 0.21)),
    (-2., [4.], [0.1], 0.02, (-0.42, 0.21)),
    (-2., [4.], [0.1], 0., (-0.4, 0.2)),
    (-2., [0.], [0.1], 0., (0., 0.)),
    (2., [20.], [0.1], 0.1, (2., 1.)),
    (-2., [20.], [0.1], 0.1, (-2., 1.)),
    (0., [1.], [0.1], 0.1, (0., 1.)),
    (0., [1.], [0.1], 0., (0., 1.)),
    (0., [0.], [0.], 0., (0., 1.)),
    (2., [4., -5.], [0.1, 0.2], 0.02, (4 * .1 + 5 * .2 + .02, (4 * .1 + 5 * .2 + .02) / 2)),   # test_scalar_multiple_clip
    (2., [], [], 0.02, (.02, .01)),                                                             # test_scalar_empty_reference
    (0., [], [], 0., (0., 1.)),
])
def test_shrink_by_references_scalars(tensor, references, relative_factors, absolute_factor, expected):
  clipped, scale = co.shrink_by_references(tensor, references, relative_factors, absolute_factor)
  _close(clipped, expected[0], rtol=1e-6, atol=1e-6)
  _close(scale, expected[1], rtol=1e-6, atol=1e-6)


@pytest.mark.parametrize("tensor,reference,absolute_factor,exp_clipped,exp_scale", [
    ([1., 1.], [1., 0.1], 0.01, [0.02, 0.02], 0.02),                       # test_tensor_clip
    ([1., 1., 0., 0.], [1., 0.1, 1., 0.], 0., [0.01, 0.01, 0., 0.], 0.01),  # test_tensor_clip_zero_absolute_factor
    ([1., 1., 0., 0.], [1., 0., 1., 0.], 0., [0., 0., 0., 0.], 0.),         # test_tensor_clip_zero_reference
    ([[1., 2.], [1., 2.]], 1., 0.1, [[0.1, 0.2], [0.1, 0.2]], 0.1),         # test_broadcast
])
def test_shrink_by_references_tensors(tensor, reference, absolute_factor, exp_clipped, exp_scale):
  clipped, scale = co.shrink_by_references(np.array(tensor), [np.array(reference)], [0.1], absolute_factor)
  _close(clipped, exp_clipped, rtol=1e-6, atol=1e-6)
  _close(scale, exp_scale, rtol=1e-6, atol=1e-6)


@pytest.mark.parametrize("relative_factors,absolute_factor,references,match", [
    ([-0.1], 0.02, [4.], "relative_factors must all be non-negative"),
    ([0.1], -0.02, [4.], "absolute_factor must be non-negative"),
    ([0.1, 0.2], 0.02, [4.], "must have the same length"),
])
def test_shrink_by_references_value_errors(relative_factors, absolute_factor, references, match):
  """clippy_adagrad.py:51-58, in the oracle and in the product (raised before anything touches a device)."""
  from recommenders_b200.experimental.optimizers import shrink_by_references
  for fn in (co.shrink_by_references, shrink_by_references):
    with pytest.raises(ValueError, match=match):
      fn(2., references, relative_factors, absolute_factor)


# ---- ClippyAdagradTest step tests (clippy_adagrad_test.py:164-303): dense [1, 2], sparse [[3, 4], [1, 2]] at index 1 ----
def _oracle_step(dense_g, sparse_g, lr, init, **kw):
  x, xa, xf = co.clippy_adagrad_dense(np.array([1., 2.]), np.full(2, init), np.array(dense_g), lr, **kw)
  s, sa, sf = co.clippy_adagrad_sparse(np.array([[3., 4.], [1., 2.]]), np.full((2, 2), init), np.array([1]),
                                        np.array([sparse_g]), lr, **kw)
  return x, xa, xf, s, sa, sf


def test_single_step_no_clip():
  lr, s0 = 0.1, 0.1
  x, xa, xf, s, sa, sf = _oracle_step([0.1, 0.15], [0.1, 0.15], lr, s0 ** 2)
  _close(x, [1.0 - lr * 0.1 / s0, 2.0 - lr * 0.15 / s0])
  _close(s, [[3.0, 4.0], [1.0 - lr * 0.1 / s0, 2.0 - lr * 0.15 / s0]])
  _close(xa, [s0 ** 2 + 0.1 ** 2, s0 ** 2 + 0.15 ** 2])
  _close(sa, [[s0 ** 2, s0 ** 2], [s0 ** 2 + 0.1 ** 2, s0 ** 2 + 0.15 ** 2]])
  _close([xf, sf], [1.0, 1.0])


@pytest.mark.parametrize("clip_accumulator_update", [False, True])
def test_single_step_clip(clip_accumulator_update):
  """test_single_step_clip and test_single_step_clip_with_accumulator."""
  lr, s0 = 0.2, 0.1
  x, xa, xf, s, sa, sf = _oracle_step([10., 10.], [10., 10.], lr, s0 ** 2, eps=0.0, var_rel=0.4, acc_rel=0.01,
                                      abs_thr=0.1, clip_accumulator_update=clip_accumulator_update)
  _close(x, [0.4, 1.4])
  _close(s, [[3.0, 4.0], [0.4, 1.4]])
  factor = 0.6 * s0 / (10.0 * lr)
  _close([xf, sf], [factor, factor])
  u = factor * 10 if clip_accumulator_update else 10.
  _close(xa, [s0 ** 2 + u ** 2] * 2)
  _close(sa, [[s0 ** 2, s0 ** 2], [s0 ** 2 + u ** 2] * 2])


def test_single_step_clip_with_standard_update():
  lr = 0.1
  x, xa, xf, s, sa, sf = _oracle_step([0.1, 0.15], [0.1, 0.15], lr, 0.0, use_standard_accumulator_update=True)
  _close(x, [1.0 - lr, 2.0 - lr])
  _close(s, [[3.0, 4.0], [1.0 - lr, 2.0 - lr]])
  _close(xa, np.square(np.float32([0.1, 0.15])))
  _close(sa, [[0., 0.], [0.1 ** 2, 0.15 ** 2]])
  _close([xf, sf], [1.0, 1.0])


def test_oracle_sums_duplicate_ids_and_skips_out_of_range():
  """The sparse rule runs on the summed row of each distinct id (duplicates in order of occurrence) and the factor is a
  minimum over the touched rows only."""
  t = np.array([[1., 2.], [3., 4.], [0., 5.]], np.float32); a = np.full_like(t, 0.1)
  g = np.array([[0.5, 0.25], [0.125, 1.], [9., 9.], [0.25, 0.5]], np.float32)
  t1, a1, f1 = co.clippy_adagrad_sparse(t, a, [0, 1, 7, 0], g, 0.3, var_rel=0.2)
  t2, a2, f2 = co.clippy_adagrad_sparse(t, a, [0, 1], np.stack([g[0] + g[3], g[1]]), 0.3, var_rel=0.2)
  assert np.array_equal(t1, t2) and np.array_equal(a1, a2) and f1 == f2 and 0 < f1 < 1
  assert np.array_equal(t1[2], t[2]) and np.array_equal(a1[2], a[2])


# ---- the public classes: construction, config and the checks that run before any kernel --------------------------------
def test_clippy_adagrad_constructor_and_config():
  from recommenders_b200.experimental.optimizers import ClippyAdagrad
  with pytest.raises(ValueError, match="cannot both be set to True"):
    ClippyAdagrad(clip_accumulator_update=True, use_standard_accumulator_update=True)
  opt = ClippyAdagrad()
  assert (opt.learning_rate, opt.initial_accumulator_value, opt.variable_relative_threshold,
          opt.accumulator_relative_threshold, opt.absolute_threshold, opt.epsilon, opt.export_clipping_factors,
          opt.clip_accumulator_update, opt.use_standard_accumulator_update) == (0.001, 0.1, 0.1, 0.0, 1e-7, 1e-7, False, False,
                                                                                 False)
  assert opt.clipping_factors == [] and opt.iterations == 0
  # clippy_adagrad_test.py:344-370, plus use_standard_accumulator_update, which the reference's get_config drops
  opt = ClippyAdagrad(learning_rate=0.1, initial_accumulator_value=0.2, variable_relative_threshold=0.3,
                      accumulator_relative_threshold=0.6, absolute_threshold=0.4, epsilon=0.5, export_clipping_factors=True,
                      use_standard_accumulator_update=True, name="clippy")
  restored = ClippyAdagrad.from_config(opt.get_config())
  for attr in ("learning_rate", "initial_accumulator_value", "variable_relative_threshold", "absolute_threshold", "epsilon",
               "export_clipping_factors", "accumulator_relative_threshold", "clip_accumulator_update",
               "use_standard_accumulator_update", "name"):
    assert getattr(restored, attr) == getattr(opt, attr), attr
  restored = ClippyAdagrad.from_config(ClippyAdagrad(clip_accumulator_update=True).get_config())
  assert restored.clip_accumulator_update and not restored.use_standard_accumulator_update


def _three_variable_module():
  m = torch.nn.Module()
  m.var1 = torch.nn.Parameter(torch.tensor([0.1, 0.2, 1.0]))
  m.var2 = torch.nn.Parameter(torch.tensor([-5.1, 0.1, 0.0]))
  m.var3 = torch.nn.Parameter(torch.tensor([-2.1, 1.3, 0.0]))
  for p, g in ((m.var1, [0.1, 0.2, 1.0]), (m.var2, [0.5, 0.0, -2.0]), (m.var3, [-0.2, 0.0, -1.0])):
    p.grad = torch.tensor(g)
  return m


def test_composite_optimizer_incorrect_inputs():
  """composite_optimizer_test.py:88-117: a variable claimed twice, or a trainable variable claimed by none, raises
  before any optimizer runs (the variables here live on the CPU, where an update would fail)."""
  from recommenders_b200 import optimizers
  from recommenders_b200.experimental.optimizers import ClippyAdagrad, CompositeOptimizer
  with pytest.raises(ValueError, match="can't be empty"):
    CompositeOptimizer([])
  m = _three_variable_module()
  before = [p.detach().clone() for p in m.parameters()]
  twice = CompositeOptimizer([(ClippyAdagrad(), lambda: [m.var1]), (optimizers.Adagrad(), lambda: [m.var1, m.var2, m.var3])])
  twice.bind(m)
  with pytest.raises(ValueError, match="should be disjoint"):
    twice.apply_gradients()
  missing = CompositeOptimizer([(ClippyAdagrad(), lambda: [m.var1]), (optimizers.Adagrad(), lambda: [m.var2])])
  missing.bind(m)
  with pytest.raises(ValueError, match="not handled by any optimizer"):
    missing.apply_gradients()
  assert all(torch.equal(a, b) for a, b in zip(before, m.parameters()))
  assert twice.optimizers[1].iterations == 0 and missing.iterations == 0
  with pytest.raises(NotImplementedError):
    missing.get_config()


def test_variable_helpers_match_adagrad_discovery():
  from recommenders_b200 import optimizers
  m = _three_variable_module()
  m.frozen = torch.nn.Parameter(torch.zeros(2), requires_grad=False)
  assert optimizers.embedding_tables(m) == []
  assert [id(p) for p in optimizers.dense_variables(m)] == [id(m.var1), id(m.var2), id(m.var3)]
  tables, dense = optimizers.split_variables([m.var2, m.var1])
  assert tables == [] and [id(p) for p in dense] == [id(m.var2), id(m.var1)]
  with pytest.raises(TypeError):
    optimizers.split_variables([3.0])
