"""NumPy oracle of K23 and K24: Philox4x32-10 and the dropout mask, bit for bit, and a float64 BatchNormalization
forward and backward (training, inference, masked rows and the moving-statistics update).  DESIGN.md §2 (A26) states
the rules."""
from __future__ import annotations

import math

import numpy as np

M0, M1 = 0xD2511F53, 0xCD9E8D57
W0, W1 = 0x9E3779B9, 0xBB67AE85
U32 = 0xFFFFFFFF


def philox4x32_10(ctr, key):
  """ctr: four uint32 arrays (or ints) of one shape, key: two.  Returns the four output words as uint32 arrays."""
  c = [np.asarray(v, dtype=np.uint64) for v in ctr]
  k0, k1 = (np.uint64(int(v) & U32) for v in key)
  for r in range(10):
    if r:
      k0, k1 = (k0 + np.uint64(W0)) & np.uint64(U32), (k1 + np.uint64(W1)) & np.uint64(U32)
    p0, p1 = np.uint64(M0) * c[0], np.uint64(M1) * c[2]
    c = [(p1 >> np.uint64(32)) ^ c[1] ^ k0, p1 & np.uint64(U32), (p0 >> np.uint64(32)) ^ c[3] ^ k1, p0 & np.uint64(U32)]
  return [v.astype(np.uint32) for v in c]


def threshold(rate: float) -> int:
  """keep <=> (word >> 8) >= threshold(rate)."""
  return int(math.ceil(float(rate) * 2.0**24))


def scale_of(rate: float) -> np.float32:
  return np.float32(1.0 / (1.0 - float(rate)))


def noise_shape_of(shape, noise_shape):
  if noise_shape is None:
    return tuple(shape)
  return tuple(s if n is None else int(n) for s, n in zip(shape, noise_shape))


def dropout_keep(noise_shape, rate: float, seed: int, call: int) -> np.ndarray:
  """bool [noise_shape]: mask element j (row-major) takes word j % 4 of Philox at counter (j // 4, call), key seed."""
  n = int(np.prod(noise_shape, dtype=np.int64))
  g = np.arange((n + 3) // 4, dtype=np.uint64)
  seed, call = int(seed) & (2**64 - 1), int(call) & (2**64 - 1)
  words = philox4x32_10((g & np.uint64(U32), g >> np.uint64(32), call & U32, call >> 32), (seed & U32, seed >> 32))
  w = np.stack(words, axis=1).reshape(-1)[:n]
  return ((w >> np.uint32(8)) >= np.uint32(threshold(rate))).reshape(noise_shape)


def dropout(x: np.ndarray, rate: float, seed: int, call: int, noise_shape=None) -> np.ndarray:
  """float32 y = keep ? x * f32(1 / (1 - rate)) : +0, the mask broadcast from the noise shape."""
  x = np.asarray(x, dtype=np.float32)
  keep = dropout_keep(noise_shape_of(x.shape, noise_shape), rate, seed, call)
  return np.where(keep, x * scale_of(rate), np.float32(0.0)).astype(np.float32)


# ---- batch normalization (float64) ---------------------------------------------------------------------------------
def _weights(x2, mask):
  return np.ones(x2.shape[0]) if mask is None else (np.asarray(mask).reshape(-1) != 0).astype(np.float64)


def batch_moments(x, mask=None):
  """(mean [d], population variance [d], n) over the rows of x [..., d] that `mask` ([...], nonzero = kept) keeps;
  n = 0 gives mean 0 and variance 0."""
  x2 = np.asarray(x, np.float64).reshape(-1, np.shape(x)[-1])
  w = _weights(x2, mask)
  n = w.sum()
  if n == 0:
    return np.zeros(x2.shape[1]), np.zeros(x2.shape[1]), 0.0
  mean = (w[:, None] * x2).sum(0) / n
  var = (w[:, None] * (x2 - mean) ** 2).sum(0) / n
  return mean, var, n


def moving_update(moving, batch, momentum: float):
  """tf-keras's _assign_moving_average: moving - (moving - batch) * f32(1 - momentum)."""
  decay = float(np.float32(1.0 - momentum))
  return np.asarray(moving, np.float64) - (np.asarray(moving, np.float64) - batch) * decay


def batch_norm_forward(x, gamma, beta, moving_mean, moving_variance, training: bool, momentum=0.99, epsilon=1e-3,
                       mask=None):
  """(y [x.shape], new moving_mean, new moving_variance); the moving statistics are unchanged at inference."""
  x = np.asarray(x, np.float64)
  d = x.shape[-1]
  x2 = x.reshape(-1, d)
  eps = float(np.float32(epsilon))
  mm, mv = np.asarray(moving_mean, np.float64), np.asarray(moving_variance, np.float64)
  if training:
    mean, var, _ = batch_moments(x2, mask)
    new_mm, new_mv = moving_update(mm, mean, momentum), moving_update(mv, var, momentum)
  else:
    mean, var, new_mm, new_mv = mm, mv, mm, mv
  xhat = (x2 - mean) / np.sqrt(var + eps)
  y = xhat * (1.0 if gamma is None else np.asarray(gamma, np.float64)) + (0.0 if beta is None else np.asarray(beta, np.float64))
  return y.reshape(x.shape), new_mm, new_mv


def batch_norm_backward(x, gamma, dy, moving_mean, moving_variance, training: bool, epsilon=1e-3, mask=None):
  """(dx, dgamma, dbeta).  dgamma = sum_rows dy xhat and dbeta = sum_rows dy over all rows; in training dx = gamma rstd
  (dy - w (S1 + xhat S2) / n), at inference dx = dy gamma rstd_mv."""
  x = np.asarray(x, np.float64)
  d = x.shape[-1]
  x2, g2 = x.reshape(-1, d), np.asarray(dy, np.float64).reshape(-1, d)
  eps = float(np.float32(epsilon))
  if training:
    mean, var, n = batch_moments(x2, mask)
  else:
    mean, var, n = np.asarray(moving_mean, np.float64), np.asarray(moving_variance, np.float64), 0.0
  rstd = 1.0 / np.sqrt(var + eps)
  xhat = (x2 - mean) * rstd
  s1, s2 = g2.sum(0), (g2 * xhat).sum(0)
  gam = 1.0 if gamma is None else np.asarray(gamma, np.float64)
  if training and n > 0:
    w = _weights(x2, mask)
    dx = gam * rstd * (g2 - w[:, None] * (s1 + xhat * s2) / n)
  else:
    dx = g2 * gam * rstd
  return dx.reshape(x.shape), s2, s1
