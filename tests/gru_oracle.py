"""float64 NumPy restatement of tf.keras.layers.GRU (reset_after=True) and of its backward through time, the reference the
K19 tests compare against.  Weights as Keras stores them: W [D, 3u], U [u, 3u], bias [2, 3u] = (b_i, b_r), columns
(z, r, h).  A masked step (mask == 0) carries h unchanged; the output sequence holds the carried h there."""
import numpy as np


def sigmoid(x):
  return 1.0 / (1.0 + np.exp(-x))


def _split(a, u):
  return a[..., :u], a[..., u:2 * u], a[..., 2 * u:]


def forward(x, W, U, bias=None, h0=None, mask=None):
  """(seq [B, T, u], h_T [B, u], cache) for x [B, T, D]."""
  x, W, U = (np.asarray(a, np.float64) for a in (x, W, U))
  B, T, _ = x.shape
  u = U.shape[0]
  b_i, b_r = (0.0, 0.0) if bias is None else np.asarray(bias, np.float64)
  h = np.zeros((B, u)) if h0 is None else np.asarray(h0, np.float64).copy()
  keep = np.ones((B, T), bool) if mask is None else np.asarray(mask) != 0
  gx = x @ W + b_i
  seq, cache = np.zeros((B, T, u)), []
  for t in range(T):
    gr = h @ U + b_r
    xz, xr, xh = _split(gx[:, t], u)
    rz, rr, rh = _split(gr, u)
    z, r = sigmoid(xz + rz), sigmoid(xr + rr)
    hh = np.tanh(xh + r * rh)
    k = keep[:, t:t + 1]
    cache.append((h, z, r, hh, rh, k))
    h = np.where(k, z * h + (1 - z) * hh, h)
    seq[:, t] = h
  return seq, h, cache


def backward(x, W, U, bias=None, h0=None, mask=None, g_seq=None, g_last=None):
  """Gradients of sum(seq * g_seq) + sum(h_T * g_last): dict of dx, dW, dU, dbias ([2, 3u], None without bias), dh0,
  and the projection's gradient dgx [B, T, 3u]."""
  x, W, U = (np.asarray(a, np.float64) for a in (x, W, U))
  B, T, D = x.shape
  u = U.shape[0]
  _, _, cache = forward(x, W, U, bias, h0, mask)
  dh = np.zeros((B, u))
  dgx, dU, db_r = np.zeros((B, T, 3 * u)), np.zeros_like(U), np.zeros(3 * u)
  for t in reversed(range(T)):
    if g_seq is not None:
      dh = dh + np.asarray(g_seq, np.float64)[:, t]
    if g_last is not None and t == T - 1:
      dh = dh + np.asarray(g_last, np.float64)
    hp, z, r, hh, rh, k = cache[t]
    dz = dh * (hp - hh) * z * (1 - z)
    dn = dh * (1 - z) * (1 - hh * hh)
    dr = dn * rh * r * (1 - r)
    dgx[:, t] = np.concatenate([dz, dr, dn], 1) * k
    dgr = np.concatenate([dz, dr, dn * r], 1) * k
    dU += hp.T @ dgr
    db_r += dgr.sum(0)
    dh = np.where(k, dh * z + dgr @ U.T, dh)
  g2 = dgx.reshape(B * T, 3 * u)
  out = {"dx": (g2 @ W.T).reshape(B, T, D), "dW": x.reshape(B * T, D).T @ g2, "dU": dU, "dh0": dh, "dgx": dgx,
         "dbias": None if bias is None else np.stack([g2.sum(0), db_r])}
  return out
