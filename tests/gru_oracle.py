"""float64 NumPy restatement of tf.keras.layers.GRU (reset_after=True) and of its backward through time, the reference the
K19 tests compare against.  Weights as Keras stores them: W [D, 3u], U [u, 3u], bias [2, 3u] = (b_i, b_r), columns
(z, r, h).  A masked step (mask == 0) carries h unchanged; the output sequence holds the carried h there.

Each direction also stands on its own, as the kernels do: `forward_gx` starts at the projection gx, `reverse` at the
tensors the forward saves (gates, h_prev), and both return first-order bounds (tests/rnn_error.py, units of 2^-24) on
the float32 kernels' error per element, built in the operation order of csrc/gru.cu."""
import numpy as np

import rnn_error as re_


def sigmoid(x):
  return 1.0 / (1.0 + np.exp(-x))


def _split(a, u):
  return a[..., :u], a[..., u:2 * u], a[..., 2 * u:]


def _keep(mask, B, T):
  return np.ones((B, T), bool) if mask is None else np.asarray(mask) != 0


def forward_gx(gx, U, b_r=None, h0=None, mask=None, bounds=True):
  """The recurrence from gx [B, T, 3u] (float64 of the given values).  Returns (out, err): out holds seq [B, T, u],
  h_T [B, u], gates [B, T, 4u] = (z, r, hh, gr_h) and h_prev [B, T, u] (what the kernel saves; gates at masked steps
  are what the step would have computed), keep [B, T]; err the bounds of seq, h_T, gates and h_prev."""
  gx, U = np.asarray(gx, np.float64), np.asarray(U, np.float64)
  B, T, _ = gx.shape
  u = U.shape[0]
  keep = _keep(mask, B, T)
  h = re_.exact(np.zeros((B, u)) if h0 is None else np.asarray(h0, np.float64))
  br = None if b_r is None else np.asarray(b_r, np.float64)
  seq, gates, hprev = (np.zeros((2, B, T, n)) for n in (u, 4 * u, u))
  for t in range(T):
    a = re_.chain(h, U, bounds)
    az, ar, ah = a[:u], a[u:2 * u], a[2 * u:]
    if br is not None:
      az, ar, ah = (re_.add(x, re_.exact(br[q * u:(q + 1) * u])) for q, x in enumerate((az, ar, ah)))
    xz, xr, xh = (re_.exact(v) for v in _split(gx[:, t], u))
    z = re_.sigmoid(re_.add(xz, az))
    r = re_.sigmoid(re_.add(xr, ar))
    hh = re_.tanh(re_.add(xh, re_.mul(r, ah)))
    hn = re_.add(re_.mul(z, h), re_.mul(re_.one_minus(z), hh))
    for dst, f in ((gates, re_.cat([z, r, hh, ah])), (hprev, h)):
      dst[0, :, t], dst[1, :, t] = f.v, f.e
    h = re_.where(keep[:, t:t + 1], hn, h)
    seq[0, :, t], seq[1, :, t] = h.v, h.e
  out = {"seq": seq[0], "h_T": h.v, "gates": gates[0], "h_prev": hprev[0], "keep": keep}
  err = {"seq": seq[1], "h_T": h.e, "gates": gates[1], "h_prev": hprev[1]}
  return out, err


def reverse(U, gates, h_prev, mask=None, g_seq=None, g_last=None, bounds=True):
  """The backward through time from the saved gates [B, T, 4u] and h_prev [B, T, u] (float64 of the given values, as
  the kernel reads them).  Returns (out, err): out holds dgx [B, T, 3u], dgr [B, T, 3u] (U's output gradient, zero at
  masked steps) and dh0 [B, u]; err the bounds of dgx and dh0."""
  U, gates, h_prev = (np.asarray(a, np.float64) for a in (U, gates, h_prev))
  B, T, u = h_prev.shape
  keep = _keep(mask, B, T)
  UT = U.T
  dh = re_.exact(np.zeros((B, u)))
  dgx, dgr = np.zeros((2, B, T, 3 * u)), np.zeros((B, T, 3 * u))
  for t in reversed(range(T)):
    d = dh
    if g_seq is not None:
      d = re_.add(d, re_.exact(np.asarray(g_seq, np.float64)[:, t]))
    if g_last is not None and t == T - 1:
      d = re_.add(d, re_.exact(np.asarray(g_last, np.float64)))
    g = gates[:, t]
    z, r, hh, grh = (re_.exact(g[:, q * u:(q + 1) * u]) for q in range(4))
    hp = re_.exact(h_prev[:, t])
    dz = re_.mul(re_.mul(d, re_.sub(hp, hh)), re_.sigmoid_grad(z))
    dhp = re_.mul(re_.mul(d, re_.one_minus(z)), re_.tanh_grad(hh))
    dr = re_.mul(re_.mul(dhp, grh), re_.sigmoid_grad(r))
    dgh = re_.mul(dhp, r)
    k = keep[:, t:t + 1]
    gr = re_.cat([dz, dr, dgh])
    gr = re_.F(gr.v * k, gr.e * k)
    dhn = re_.add(re_.mul(d, z), re_.chain(gr, UT, bounds))
    gx_ = re_.cat([dz, dr, dhp])
    dgx[0, :, t], dgx[1, :, t] = gx_.v * k, gx_.e * k
    dgr[:, t] = gr.v
    dh = re_.where(k, dhn, d)
  return {"dgx": dgx[0], "dgr": dgr, "dh0": dh.v}, {"dgx": dgx[1], "dh0": dh.e}


def forward(x, W, U, bias=None, h0=None, mask=None):
  """(seq [B, T, u], h_T [B, u], cache) for x [B, T, D]; cache is forward_gx's output."""
  x, W = np.asarray(x, np.float64), np.asarray(W, np.float64)
  b_i, b_r = (0.0, None) if bias is None else np.asarray(bias, np.float64)
  out, _ = forward_gx(x @ W + b_i, U, b_r, h0, mask, bounds=False)
  return out["seq"], out["h_T"], out


def backward(x, W, U, bias=None, h0=None, mask=None, g_seq=None, g_last=None):
  """Gradients of sum(seq * g_seq) + sum(h_T * g_last): dict of dx, dW, dU, dbias ([2, 3u], None without bias), dh0,
  and the projection's gradient dgx [B, T, 3u]."""
  x, W = np.asarray(x, np.float64), np.asarray(W, np.float64)
  B, T, D = x.shape
  _, _, c = forward(x, W, U, bias, h0, mask)
  r, _ = reverse(U, c["gates"], c["h_prev"], mask, g_seq, g_last, bounds=False)
  u = c["h_prev"].shape[-1]
  g2, gr2 = r["dgx"].reshape(B * T, 3 * u), r["dgr"].reshape(B * T, 3 * u)
  return {"dx": (g2 @ W.T).reshape(B, T, D), "dW": x.reshape(B * T, D).T @ g2,
          "dU": c["h_prev"].reshape(B * T, u).T @ gr2, "dh0": r["dh0"], "dgx": r["dgx"],
          "dbias": None if bias is None else np.stack([g2.sum(0), gr2.sum(0)])}
