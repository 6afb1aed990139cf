"""CPU oracle of FTRL-Proximal (recommenders_b200.optimizers.Ftrl: tf-keras's legacy optimizer_v2/ftrl.py rules, which
call TF's ApplyFtrl / ApplyFtrlV2 and their sparse forms), used by the optimizer tests.

TEST INFRASTRUCTURE ONLY, like oracle/: the product (recommenders_b200/) never imports it.  The fp32 functions state the
update rule step by step in NumPy float32: every NumPy float32 add, multiply, divide and sqrt is one correctly rounded
IEEE operation, and separate ufunc calls are never contracted into an FMA.  That makes them the bit-exact bar of the K12
kernels (csrc/ftrl.cu).

Per call, on the host:  l2a = l2 + beta / (2*lr)            fp32, one operation at a time
Power term:  P(x) = sqrt(x)                                 when lr_power == -0.5 (fp32)
             P(x) = f32(pow(f64(x), -f64(lr_power)))        otherwise: float64 pow, rounded once
Per element, with g the gradient:
  gs   = g + (2*l2_shrinkage)*var   if l2_shrinkage > 0, else g
  na   = acc + g*g
  lin' = lin + (gs - ((P(na) - P(acc)) / lr)*var)
  y    = P(na)/lr + 2*l2a
  var' = (copysign(l1, lin') - lin') / y   if |lin'| > l1, else +0
  acc' = na
Sparse gradients: duplicate ids are summed first, in order of occurrence; out-of-range ids are skipped; only the touched
rows change.
"""
from __future__ import annotations

import numpy as np

from clippy_oracle import _summed_rows

F32 = np.float32


def l2a(l2: float, beta: float, lr: float) -> np.float32:
  """tf-keras's adjusted l2 strength: l2 + beta / (2*lr), in fp32."""
  return F32(l2) + F32(beta) / (F32(2) * F32(lr))


def power(x, lr_power: float):
  """P(x) of the element rule on a float32 array."""
  if F32(lr_power) == F32(-0.5):
    return np.sqrt(x)
  return np.power(np.asarray(x, np.float64), -np.float64(F32(lr_power))).astype(np.float32)


def _rule(var, acc, lin, g, lr, lr_power, l1, l2, l2_shrinkage, beta):
  lr32, l1, s = F32(lr), F32(l1), F32(l2_shrinkage)
  two_l2a = F32(2) * l2a(l2, beta, lr)
  gs = g + (F32(2) * s) * var if s > 0 else g
  na = acc + g * g
  pn, pa = power(na, lr_power), power(acc, lr_power)
  lin1 = lin + (gs - ((pn - pa) / lr32) * var)
  with np.errstate(divide="ignore", invalid="ignore"):
    y = pn / lr32 + two_l2a
    var1 = np.where(np.abs(lin1) > l1, (np.copysign(l1, lin1) - lin1) / y, F32(0)).astype(np.float32)
  return var1, na, lin1


def ftrl_dense(var, acc, lin, grad, lr: float = 0.001, lr_power: float = -0.5, l1: float = 0.0, l2: float = 0.0,
               l2_shrinkage: float = 0.0, beta: float = 0.0):
  """One step of the element rule on a dense variable; returns (var, acc, lin) as new float32 arrays."""
  x, a, z, g = (np.array(t, np.float32) for t in (var, acc, lin, grad))
  return _rule(x, a, z, g, lr, lr_power, l1, l2, l2_shrinkage, beta)


def ftrl_sparse(table, acc, lin, ids, grad_rows, lr: float = 0.001, lr_power: float = -0.5, l1: float = 0.0,
                l2: float = 0.0, l2_shrinkage: float = 0.0, beta: float = 0.0):
  """One step on an embedding table: the element rule on the touched rows only; returns (table, acc, lin) as new float32
  arrays."""
  x, a, z = (np.array(t, np.float32) for t in (table, acc, lin))
  if not np.size(ids):
    return x, a, z
  heads, g = _summed_rows(ids, grad_rows, x.shape[0])
  x[heads], a[heads], z[heads] = _rule(x[heads], a[heads], z[heads], g, lr, lr_power, l1, l2, l2_shrinkage, beta)
  return x, a, z


def ftrl_textbook(var, acc, lin, grad, lr: float, lr_power: float = -0.5, l1: float = 0.0, l2: float = 0.0,
                  l2_shrinkage: float = 0.0, beta: float = 0.0):
  """The same rule in float64, with P(x) = x^(-lr_power) for every lr_power (McMahan et al. 2013, Algorithm 1, with
  TF's learning-rate power and shrinkage)."""
  x, a, z, g = (np.asarray(t, np.float64) for t in (var, acc, lin, grad))
  l2 = l2 + beta / (2.0 * lr)
  gs = g + 2.0 * l2_shrinkage * x if l2_shrinkage > 0 else g
  na = a + g * g
  pn, pa = na ** -lr_power, a ** -lr_power
  z = z + gs - (pn - pa) / lr * x
  y = pn / lr + 2.0 * l2
  x = np.where(np.abs(z) > l1, (np.sign(z) * l1 - z) / y, 0.0)
  return x, na, z
