"""Float64 NumPy restatement of K27 (layers.Conv1D): Keras's padding geometry, the im2col matrix, the forward with every
activation, the backward of the fused linear part, and the per-element bars of the GPU tests."""
import math

import numpy as np

PADDINGS = ("valid", "same", "causal")


def geometry(T, k, s=1, d=1, padding="valid"):
  """(T_out, left pad, right pad) of tf-keras's Conv1D, or None where "valid" leaves no output step."""
  span = d * (k - 1) + 1
  if padding == "valid":
    return ((T - span) // s + 1, 0, 0) if T >= span else None
  T_out = -(-T // s)
  if padding == "same":
    total = max((T_out - 1) * s + span - T, 0)
    return T_out, total // 2, total - total // 2
  return T_out, span - 1, 0


def col_index(T, k, s, d, p, T_out):
  """[T_out, k] time index t_out s + j d - p read by window t_out at tap j (outside [0, T): no read)."""
  return np.arange(T_out)[:, None] * s + np.arange(k)[None, :] * d - p


def im2col(x, k, s, d, p, T_out):
  """col [B T_out, k C] with col[(b, t), j C + c] = x[b, t s + j d - p, c], 0 outside the sequence."""
  B, T, C = x.shape
  idx = col_index(T, k, s, d, p, T_out)
  ok = (idx >= 0) & (idx < T)
  g = np.asarray(x, np.float64)[:, np.clip(idx, 0, T - 1), :] * ok[None, :, :, None]   # [B, T_out, k, C]
  return g.reshape(B * T_out, k * C)


def col2im(dcol, B, T, C, k, s, d, p, T_out):
  """dx [B, T, C]: the adjoint of im2col."""
  idx = col_index(T, k, s, d, p, T_out)
  g = np.asarray(dcol, np.float64).reshape(B, T_out, k, C)
  dx = np.zeros((B, T, C))
  for j in range(k):
    for to in range(T_out):
      t = idx[to, j]
      if 0 <= t < T:
        dx[:, t, :] += g[:, to, j, :]
  return dx


def _gelu(z):
  return 0.5 * z * (1.0 + np.vectorize(math.erf)(z / math.sqrt(2.0)))


ACTIVATIONS = {
    None: lambda z: z, "linear": lambda z: z, "relu": lambda z: np.maximum(z, 0.0),
    "sigmoid": lambda z: 1.0 / (1.0 + np.exp(-z)), "tanh": np.tanh,
    "swish": lambda z: z / (1.0 + np.exp(-z)), "silu": lambda z: z / (1.0 + np.exp(-z)), "gelu": _gelu,
}


def forward(x, W, b, s=1, d=1, padding="valid", activation=None):
  """(z, y, col): z = the linear part [B, T_out, F], y = act(z), col the im2col matrix."""
  B, T, C = x.shape
  k, _, F = W.shape
  T_out, p, _ = geometry(T, k, s, d, padding)
  col = im2col(x, k, s, d, p, T_out)
  z = col @ np.asarray(W, np.float64).reshape(k * C, F)
  if b is not None:
    z = z + np.asarray(b, np.float64)[None, :]
  z = z.reshape(B, T_out, F)
  return z, ACTIVATIONS[activation](z), col


def backward(x, W, dz, s=1, d=1, padding="valid"):
  """(dx, dW, dbias) of the linear part from dz [B, T_out, F]."""
  B, T, C = x.shape
  k, _, F = W.shape
  T_out, p, _ = geometry(T, k, s, d, padding)
  col = im2col(x, k, s, d, p, T_out)
  dz2 = np.asarray(dz, np.float64).reshape(B * T_out, F)
  dcol = dz2 @ np.asarray(W, np.float64).reshape(k * C, F).T
  dx = col2im(dcol, B, T, C, k, s, d, p, T_out)
  return dx, (col.T @ dz2).reshape(k, C, F), dz2.sum(0)


def ebar(A, Bm, amax_a=None, amax_b=None):
  """Bar (E) of the split-GEMM edge tests for A [M, K] . B [K, N]: 1e-5 (|A| |B|) + 2^-36 (amax_A sum_k |B| + amax_B sum_k
  |A|).  amax_a / amax_b override the operands' max |element|: the rescale of a gathered im2col operand is taken from
  max |x|, which bounds max |col|."""
  Af, Bf = np.abs(A), np.abs(Bm)
  aa = Af.max() if amax_a is None else amax_a
  ab = Bf.max() if amax_b is None else amax_b
  return 1e-5 * (Af @ Bf) + 2.0 ** -36 * (aa * Bf.sum(0)[None, :] + ab * Af.sum(1)[:, None])
