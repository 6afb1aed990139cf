"""CPU oracle of Adam (recommenders_b200.optimizers.Adam, tf-keras's legacy optimizer_v2/adam.py rules), used by the
optimizer tests.

TEST INFRASTRUCTURE ONLY, like oracle/: the product (recommenders_b200/) never imports it.  The fp32 functions state the
update rules step by step in NumPy float32: every NumPy float32 add, multiply, divide and sqrt is one correctly rounded
IEEE operation, and separate ufunc calls are never contracted into an FMA.  That makes them the bit-exact bar of the K10
kernels (csrc/adam.cu).

Per step, with t = iterations + 1:
  alpha = f32(lr * sqrt(1 - b2^t) / (1 - b1^t))     float64 from the fp32-rounded lr, b1, b2, rounded once
  omb1 = 1 - b1 ; omb2 = 1 - b2                     fp32
  dense:           m' = m + (g - m)*omb1 ;  v' = v + (g*g - v)*omb2 ;  var' = var - (m'*alpha) / (sqrt(v') + eps)
  sparse touched:  m' = m*b1 + g*omb1    ;  v' = v*b2 + (g*g)*omb2
  sparse other:    m' = m*b1             ;  v' = v*b2                 (lazy: other rows unchanged)
  sparse rows updated:  var' = var - (alpha*m') / (sqrt(v') + eps)
Sparse gradients: duplicate ids are summed first, in order of occurrence; out-of-range ids are skipped.
"""
from __future__ import annotations

import math

import numpy as np

from clippy_oracle import _summed_rows

F32 = np.float32


def alpha(lr: float, beta_1: float, beta_2: float, t: int) -> np.float32:
  lr, b1, b2 = (float(F32(x)) for x in (lr, beta_1, beta_2))
  return F32(lr * math.sqrt(1.0 - b2 ** t) / (1.0 - b1 ** t))


def _scalars(beta_1, beta_2, epsilon):
  b1, b2 = F32(beta_1), F32(beta_2)
  return b1, b2, F32(1) - b1, F32(1) - b2, F32(epsilon)


def _var(var, m1, v1, a, eps):
  return var - (a * m1) / (np.sqrt(v1) + eps)


def adam_dense(var, m, v, grad, lr: float, t: int, beta_1: float = 0.9, beta_2: float = 0.999, epsilon: float = 1e-7):
  """Step t of the dense rule on one variable; returns (var, m, v) as new float32 arrays."""
  x, m, v, g = (np.array(a, np.float32) for a in (var, m, v, grad))
  b1, b2, omb1, omb2, eps = _scalars(beta_1, beta_2, epsilon)
  a = alpha(lr, beta_1, beta_2, t)
  m1 = m + (g - m) * omb1
  v1 = v + (g * g - v) * omb2
  return x - (m1 * a) / (np.sqrt(v1) + eps), m1, v1


def adam_sparse(table, m, v, ids, grad_rows, lr: float, t: int, beta_1: float = 0.9, beta_2: float = 0.999,
                epsilon: float = 1e-7, lazy: bool = False):
  """Step t of the sparse rule on one embedding table; returns (table, m, v) as new float32 arrays."""
  x, m, v = (np.array(a, np.float32) for a in (table, m, v))
  b1, b2, omb1, omb2, eps = _scalars(beta_1, beta_2, epsilon)
  a = alpha(lr, beta_1, beta_2, t)
  if np.size(ids):
    heads, g = _summed_rows(ids, grad_rows, x.shape[0])
  else:
    heads, g = np.zeros(0, np.int64), np.zeros((0, x.shape[1]), np.float32)
  touched_m = m[heads] * b1 + g * omb1
  touched_v = v[heads] * b2 + (g * g) * omb2
  if lazy:
    m[heads], v[heads] = touched_m, touched_v
    x[heads] = _var(x[heads], touched_m, touched_v, a, eps)
    return x, m, v
  m, v = m * b1, v * b2
  m[heads], v[heads] = touched_m, touched_v
  return _var(x, m, v, a, eps), m, v


def adam_textbook(var, m, v, grad, lr: float, t: int, beta_1: float = 0.9, beta_2: float = 0.999,
                  epsilon: float = 1e-7):
  """TF's adam_update_numpy in float64: m = b1*m + (1-b1)*g ; v = b2*v + (1-b2)*g^2 ;
  var -= lr_t * m / (sqrt(v) + eps), lr_t = lr * sqrt(1 - b2^t) / (1 - b1^t)."""
  x, m, v, g = (np.asarray(a, np.float64) for a in (var, m, v, grad))
  lr_t = lr * math.sqrt(1 - beta_2 ** t) / (1 - beta_1 ** t)
  m = beta_1 * m + (1 - beta_1) * g
  v = beta_2 * v + (1 - beta_2) * g * g
  return x - lr_t * m / (np.sqrt(v) + epsilon), m, v
