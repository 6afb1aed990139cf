"""CPU oracle of ClippyAdagrad (experimental/optimizers/clippy_adagrad.py), used by the optimizer tests.

TEST INFRASTRUCTURE ONLY, like oracle/: the product (recommenders_b200/) never imports it.  Paths are relative to
tensorflow_recommenders/.  The fp32 functions state the update rule step by step in NumPy float32: every NumPy float32 add,
multiply, divide and sqrt is one correctly rounded IEEE operation, and separate ufunc calls are never contracted into an
FMA.  That makes them the bit-exact bar of the K7 kernels (csrc/clippy_adagrad.cu).  `shrink_by_references` is a float64
restatement, pinned by the reference's ClipByReferenceTest.

The rule, per touched element (update_step :188-254, shrink_by_references :21-70):
  a1    = standard ? a + g*g : a                       :197-203 (scatter_add / assign_add of square(grad))
  p     = 1 / sqrt(a1 + eps)                           :219 tf.math.rsqrt: rounded sqrt, then rounded divide
  delta = (lr * g) * p                                 :220
  m     = (abs_thr + |v| * var_rel) + |p| * acc_rel    :59-62 sum(..., start=absolute_factor), references [v, p]
  s     = delta == 0 ? 1 : m / |delta|                 :67-68 where(tensor == 0, 1, divide_no_nan(...))
  scale = min(1, min_i s_i)                            :69; NaN ratios do not lower it (fmin; not defined there)
  v'    = v - delta * scale                            :70 tensor * scale, :251-254 scatter_sub / assign_sub
  a'    = standard ? a1 : a + u*u,  u = clip ? g * scale : g      :232-249
Thresholds of -0.0 are taken as +0.0.  Sparse gradients: duplicate ids are summed first, in order of occurrence (tf-keras
deduplicates IndexedSlices; "parity unpinned", DESIGN.md section 2); out-of-range ids are skipped; the minimum runs over
the touched rows only.
"""
from __future__ import annotations

import numpy as np

F32 = np.float32


def _rule(lr, eps, var_rel, acc_rel, abs_thr):
  # -0.0 + 0.0 = +0.0 in round-to-nearest
  return F32(lr), F32(eps), F32(var_rel) + F32(0), F32(acc_rel) + F32(0), F32(abs_thr) + F32(0)


def _delta(g, a, lr, eps, standard):
  a1 = a + g * g if standard else a
  p = F32(1) / np.sqrt(a1 + eps)
  return (lr * g) * p, a1, p


def _factor(g, v, a, lr, eps, var_rel, acc_rel, abs_thr, standard) -> np.float32:
  delta, _, p = _delta(g, a, lr, eps, standard)
  m = (abs_thr + np.abs(v) * var_rel) + np.abs(p) * acc_rel
  with np.errstate(divide="ignore", invalid="ignore"):
    s = np.where(delta == 0, F32(1), m / np.abs(delta)).astype(np.float32)
  return F32(np.fmin(F32(1), np.fmin.reduce(s, initial=F32(1), axis=None)))


def _apply(g, v, a, scale, lr, eps, standard, clip):
  delta, a1, _ = _delta(g, a, lr, eps, standard)
  v_new = v - delta * scale
  if standard:
    return v_new, a1
  u = g * scale if clip else g
  return v_new, a + u * u


def clippy_adagrad_dense(var, accum, grad, lr: float, eps: float = 1e-7, var_rel: float = 0.1, acc_rel: float = 0.0,
                         abs_thr: float = 1e-7, clip_accumulator_update: bool = False,
                         use_standard_accumulator_update: bool = False):
  """ClippyAdagrad.update_step on a dense gradient, one variable; returns (var, accum, clipping_factor) as new arrays."""
  v = np.array(var, np.float32); a = np.array(accum, np.float32); g = np.array(grad, np.float32)
  assert v.shape == a.shape == g.shape
  lr, eps, var_rel, acc_rel, abs_thr = _rule(lr, eps, var_rel, acc_rel, abs_thr)
  scale = _factor(g, v, a, lr, eps, var_rel, acc_rel, abs_thr, use_standard_accumulator_update)
  v, a = _apply(g, v, a, scale, lr, eps, use_standard_accumulator_update, clip_accumulator_update)
  return v, a, scale


def _summed_rows(ids, grad, rows):
  """(distinct in-range ids, their gradient rows summed in order of occurrence)."""
  ids = np.asarray(ids, np.int64).reshape(-1)
  grad = np.asarray(grad, np.float32).reshape(ids.shape[0], -1)
  pos = np.flatnonzero((ids >= 0) & (ids < rows))
  order = pos[np.argsort(ids[pos], kind="stable")]          # grouped by id, positions ascending
  sid = ids[order]
  starts = np.flatnonzero(np.r_[True, sid[1:] != sid[:-1]]) if sid.size else np.zeros(0, np.int64)
  counts = np.diff(np.r_[starts, sid.size])
  sums = grad[order[starts]].copy()
  for k in range(1, int(counts.max()) if counts.size else 0):
    m = counts > k
    sums[m] = sums[m] + grad[order[starts[m] + k]]
  return sid[starts], sums


def clippy_adagrad_sparse(table, accum, ids, grad_rows, lr: float, eps: float = 1e-7, var_rel: float = 0.1,
                          acc_rel: float = 0.0, abs_thr: float = 1e-7, clip_accumulator_update: bool = False,
                          use_standard_accumulator_update: bool = False):
  """ClippyAdagrad.update_step on IndexedSlices (one embedding table); returns (table, accum, clipping_factor) as new
  arrays."""
  t = np.array(table, np.float32); a = np.array(accum, np.float32)
  heads, g = _summed_rows(ids, grad_rows, t.shape[0])
  lr, eps, var_rel, acc_rel, abs_thr = _rule(lr, eps, var_rel, acc_rel, abs_thr)
  scale = _factor(g, t[heads], a[heads], lr, eps, var_rel, acc_rel, abs_thr, use_standard_accumulator_update)
  t[heads], a[heads] = _apply(g, t[heads], a[heads], scale, lr, eps, use_standard_accumulator_update,
                              clip_accumulator_update)
  return t, a, scale


def shrink_by_references(tensor, references, relative_factors, absolute_factor):
  """shrink_by_references (clippy_adagrad.py:21-70) in float64: (tensor * scale, scale)."""
  if any(f < 0 for f in relative_factors):
    raise ValueError("relative_factors must all be non-negative.")
  if absolute_factor < 0:
    raise ValueError("absolute_factor must be non-negative.")
  if len(references) != len(relative_factors):
    raise ValueError("references and relative_factors must have the same length. "
                     f"Instead they are {len(references)} and {len(relative_factors)}.")
  t = np.asarray(tensor, np.float64)
  max_delta = np.float64(absolute_factor)
  for r, f in zip(references, relative_factors):
    max_delta = max_delta + np.abs(np.asarray(r, np.float64)) * f
  max_delta = np.broadcast_to(max_delta, np.broadcast_shapes(np.shape(max_delta), t.shape))
  at = np.broadcast_to(np.abs(t), max_delta.shape)
  with np.errstate(divide="ignore", invalid="ignore"):
    per = np.where(at == 0.0, 1.0, max_delta / np.where(at == 0.0, 1.0, at))
  scale = min(1.0, float(per.min())) if per.size else 1.0
  return t * scale, scale
