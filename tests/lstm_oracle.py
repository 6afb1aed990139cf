"""float64 NumPy restatement of tf.keras.layers.LSTM (TF2 defaults) and of its backward through time, the reference the
K20 tests compare against.  Weights as Keras stores them: W [D, 4u], U [u, 4u], bias [4u], columns (i, f, c, o).  A
masked step (mask == 0) carries h and c unchanged; the output sequence holds the carried h there."""
import numpy as np


def sigmoid(x):
  return 1.0 / (1.0 + np.exp(-x))


def _split(a, u):
  return a[..., :u], a[..., u:2 * u], a[..., 2 * u:3 * u], a[..., 3 * u:]


def forward(x, W, U, bias=None, h0=None, c0=None, mask=None):
  """(seq [B, T, u], h_T [B, u], c_T [B, u], cache) for x [B, T, D]."""
  x, W, U = (np.asarray(a, np.float64) for a in (x, W, U))
  B, T, _ = x.shape
  u = U.shape[0]
  b = 0.0 if bias is None else np.asarray(bias, np.float64)
  h = np.zeros((B, u)) if h0 is None else np.asarray(h0, np.float64).copy()
  c = np.zeros((B, u)) if c0 is None else np.asarray(c0, np.float64).copy()
  keep = np.ones((B, T), bool) if mask is None else np.asarray(mask) != 0
  gx = x @ W + b
  seq, cache = np.zeros((B, T, u)), []
  for t in range(T):
    zi, zf, zc, zo = _split(gx[:, t] + h @ U, u)
    i, f, g, o = sigmoid(zi), sigmoid(zf), np.tanh(zc), sigmoid(zo)
    cn = f * c + i * g
    k = keep[:, t:t + 1]
    cache.append((h, c, i, f, g, o, cn, k))
    h = np.where(k, o * np.tanh(cn), h)
    c = np.where(k, cn, c)
    seq[:, t] = h
  return seq, h, c, cache


def backward(x, W, U, bias=None, h0=None, c0=None, mask=None, g_seq=None, g_h=None, g_c=None):
  """Gradients of sum(seq * g_seq) + sum(h_T * g_h) + sum(c_T * g_c): dict of dx, dW, dU, dbias ([4u], None without
  bias), dh0, dc0, and the projection's gradient dz [B, T, 4u]."""
  x, W, U = (np.asarray(a, np.float64) for a in (x, W, U))
  B, T, D = x.shape
  u = U.shape[0]
  _, _, _, cache = forward(x, W, U, bias, h0, c0, mask)
  dh, dc = np.zeros((B, u)), np.zeros((B, u))
  dz, dU = np.zeros((B, T, 4 * u)), np.zeros_like(U)
  for t in reversed(range(T)):
    if g_seq is not None:
      dh = dh + np.asarray(g_seq, np.float64)[:, t]
    if t == T - 1:
      if g_h is not None:
        dh = dh + np.asarray(g_h, np.float64)
      if g_c is not None:
        dc = dc + np.asarray(g_c, np.float64)
    hp, cp, i, f, g, o, cn, k = cache[t]
    tc = np.tanh(cn)
    do = dh * tc * o * (1 - o)
    dct = dc + dh * o * (1 - tc * tc)
    di = dct * g * i * (1 - i)
    df = dct * cp * f * (1 - f)
    dg = dct * i * (1 - g * g)
    dzt = np.concatenate([di, df, dg, do], 1) * k
    dz[:, t] = dzt
    dU += hp.T @ dzt
    dh = np.where(k, dzt @ U.T, dh)
    dc = np.where(k, dct * f, dc)
  z2 = dz.reshape(B * T, 4 * u)
  return {"dx": (z2 @ W.T).reshape(B, T, D), "dW": x.reshape(B * T, D).T @ z2, "dU": dU, "dh0": dh, "dc0": dc,
          "dz": dz, "dbias": None if bias is None else z2.sum(0)}
