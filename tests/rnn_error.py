"""First-order rounding-error algebra for the float32 recurrence kernels (csrc/rnn.cuh, gru.cu, lstm.cu), shared by
tests/gru_oracle.py and tests/lstm_oracle.py.

A value is a pair (v, e): v the float64 value of the exact operation, e a bound on |float32 result - v| in units of
u_r = 2^-24, to first order.  Every float32 operation adds the rounding of its result (u_r |v|); expf and tanhf add
their 2-ulp maximum error from the CUDA Math API documentation (2 ulp <= 4 u_r |y| for a normal result); and every
operation whose result lies below 2^-126 adds one subnormal step, 2^-149 absolute (TINY in units of u_r), as
attention_oracle.core_error_bounds does.  Forms the compiler may contract to fmaf (a*b + c) round once fewer, so the
bounds hold either way."""
import numpy as np

U_R = 2.0 ** -24
TINY = 2.0 ** -125            # 2^-149 in units of u_r
SUB = 2.0 ** -126             # the smallest normal float32
EXPF_OVERFLOW = 88.72283935546875   # expf(x) is +inf above this (float32 log(FLT_MAX))


def _tiny(v):
  return TINY * (np.abs(v) < SUB)


class F:
  """(v, e): float64 value and its first-order float32 error bound in units of u_r."""
  __slots__ = ("v", "e")

  def __init__(self, v, e=None):
    self.v = np.asarray(v, np.float64)
    self.e = np.zeros(self.v.shape) if e is None else e

  def __getitem__(self, i):
    return F(self.v[..., i], self.e[..., i])


def exact(v):
  return F(v)


def add(a, b):
  v = a.v + b.v
  return F(v, a.e + b.e + np.abs(v) + _tiny(v))


def sub(a, b):
  v = a.v - b.v
  return F(v, a.e + b.e + np.abs(v) + _tiny(v))


def mul(a, b):
  v = a.v * b.v
  return F(v, np.abs(b.v) * a.e + np.abs(a.v) * b.e + np.abs(v) + _tiny(v))


def one_minus(a):
  v = 1.0 - a.v
  return F(v, a.e + np.abs(v) + _tiny(v))


def sigmoid(a):
  """1 / (1 + expf(-x)): expf (2 ulp, and the propagated error of x), the add and the correctly rounded division.  Where
  expf(-x) overflows the kernel's result is 0 and the error is the value itself."""
  with np.errstate(over="ignore"):
    s = 1.0 / (1.0 + np.exp(-a.v))
  e = s * (1.0 - s) * (a.e + 4.0) + 2.0 * s + 3 * _tiny(s)
  e = e + np.where(-a.v > EXPF_OVERFLOW, s / U_R, 0.0)
  return F(s, e)


def tanh(a):
  """tanhf: 2 ulp plus the propagated error of x."""
  y = np.tanh(a.v)
  return F(y, (1.0 - y * y) * a.e + 4.0 * np.abs(y) + 2 * _tiny(y))


def sigmoid_grad(s):
  """s (1 - s) from a saved sigmoid output."""
  return mul(s, one_minus(s))


def tanh_grad(y):
  """1 - y^2 from a saved tanh output."""
  return one_minus(mul(y, y))


def where(k, a, b):
  return F(np.where(k, a.v, b.v), np.where(k, a.e, b.e))


def cat(parts):
  return F(np.concatenate([p.v for p in parts], -1), np.concatenate([p.e for p in parts], -1))


def chain(x, W, bounds=True):
  """The fmaf chain acc = sum_k x[:, k] W[k] over k ascending from +0.0f (x [B, n] with its error, W [n, m] exact):
  each fmaf rounds once, by u_r times its partial sum, so the chain's own error is sum_i |s_i| over the partial sums
  s_i in that order; the error carried in on x adds |x error| . |W|.  bounds=False: the value alone."""
  if not bounds:
    return F(x.v @ W)
  B, n = x.v.shape
  m = W.shape[1]
  s = np.zeros((B, m))
  run = np.zeros((B, m))
  tiny = np.zeros((B, m))
  step = max(1, (1 << 21) // max(1, B * m))
  for k0 in range(0, n, step):
    p = np.cumsum(x.v[:, k0:k0 + step, None] * W[None, k0:k0 + step], axis=1) + s[:, None]
    run += np.abs(p).sum(1)
    tiny += (np.abs(p) < SUB).sum(1)
    s = p[:, -1]
  return F(s, run + x.e @ np.abs(W) + TINY * tiny)


def bar(e):
  """The GPU bar for an error bound e: 2 u_r e."""
  return 2.0 * U_R * e
