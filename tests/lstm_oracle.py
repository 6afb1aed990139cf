"""float64 NumPy restatement of tf.keras.layers.LSTM (TF2 defaults) and of its backward through time, the reference the
K20 tests compare against.  Weights as Keras stores them: W [D, 4u], U [u, 4u], bias [4u], columns (i, f, c, o).  A
masked step (mask == 0) carries h and c unchanged; the output sequence holds the carried h there.

Each direction also stands on its own, as the kernels do: `forward_gx` starts at the projection gx, `reverse` at the
tensors the forward saves (gates, c_seq) and c0, and both return first-order bounds (tests/rnn_error.py, units of
2^-24) on the float32 kernels' error per element, built in the operation order of csrc/lstm.cu."""
import numpy as np

import rnn_error as re_


def sigmoid(x):
  return 1.0 / (1.0 + np.exp(-x))


def _keep(mask, B, T):
  return np.ones((B, T), bool) if mask is None else np.asarray(mask) != 0


def forward_gx(gx, U, h0=None, c0=None, mask=None, bounds=True):
  """The recurrence from gx [B, T, 4u] (float64 of the given values).  Returns (out, err): out holds seq [B, T, u],
  h_T and c_T [B, u], gates [B, T, 4u] = (i, f, g, o), c_seq [B, T, u] (every c_t) and h_prev [B, T, u] (gates at
  masked steps are what the step would have computed), keep [B, T]; err the bounds of all but keep."""
  gx, U = np.asarray(gx, np.float64), np.asarray(U, np.float64)
  B, T, _ = gx.shape
  u = U.shape[0]
  keep = _keep(mask, B, T)
  h = re_.exact(np.zeros((B, u)) if h0 is None else np.asarray(h0, np.float64))
  c = re_.exact(np.zeros((B, u)) if c0 is None else np.asarray(c0, np.float64))
  seq, gates, cseq, hprev = (np.zeros((2, B, T, n)) for n in (u, 4 * u, u, u))
  for t in range(T):
    a = re_.chain(h, U, bounds)
    pre = [re_.add(re_.exact(gx[:, t, q * u:(q + 1) * u]), a[q * u:(q + 1) * u]) for q in range(4)]
    i, f, g, o = re_.sigmoid(pre[0]), re_.sigmoid(pre[1]), re_.tanh(pre[2]), re_.sigmoid(pre[3])
    cn = re_.add(re_.mul(f, c), re_.mul(i, g))
    hn = re_.mul(o, re_.tanh(cn))
    k = keep[:, t:t + 1]
    gates[0, :, t], gates[1, :, t] = re_.cat([i, f, g, o]).v, re_.cat([i, f, g, o]).e
    hprev[0, :, t], hprev[1, :, t] = h.v, h.e
    h, c = re_.where(k, hn, h), re_.where(k, cn, c)
    seq[0, :, t], seq[1, :, t] = h.v, h.e
    cseq[0, :, t], cseq[1, :, t] = c.v, c.e
  out = {"seq": seq[0], "h_T": h.v, "c_T": c.v, "gates": gates[0], "c_seq": cseq[0], "h_prev": hprev[0], "keep": keep}
  err = {"seq": seq[1], "h_T": h.e, "c_T": c.e, "gates": gates[1], "c_seq": cseq[1], "h_prev": hprev[1]}
  return out, err


def reverse(U, gates, c_seq, c0=None, mask=None, g_seq=None, g_h=None, g_c=None, bounds=True):
  """The backward through time from the saved gates [B, T, 4u], c_seq [B, T, u] and c0 (float64 of the given values, as
  the kernel reads them).  Returns (out, err): out holds dz [B, T, 4u] (zero at masked steps), dh0 and dc0 [B, u]; err
  their bounds."""
  U, gates, c_seq = (np.asarray(a, np.float64) for a in (U, gates, c_seq))
  B, T, u = c_seq.shape
  keep = _keep(mask, B, T)
  UT = U.T
  c0 = np.zeros((B, u)) if c0 is None else np.asarray(c0, np.float64)
  dh, dc = re_.exact(np.zeros((B, u))), re_.exact(np.zeros((B, u)))
  dz = np.zeros((2, B, T, 4 * u))
  for t in reversed(range(T)):
    d = dh
    if g_seq is not None:
      d = re_.add(d, re_.exact(np.asarray(g_seq, np.float64)[:, t]))
    if t == T - 1:
      if g_h is not None:
        d = re_.add(d, re_.exact(np.asarray(g_h, np.float64)))
      if g_c is not None:
        dc = re_.add(dc, re_.exact(np.asarray(g_c, np.float64)))
    g = gates[:, t]
    ig, fg, gg, og = (re_.exact(g[:, q * u:(q + 1) * u]) for q in range(4))
    cp = re_.exact(c_seq[:, t - 1] if t > 0 else c0)
    tc = re_.tanh(re_.exact(c_seq[:, t]))
    dout = re_.mul(re_.mul(d, tc), re_.sigmoid_grad(og))
    dct = re_.add(dc, re_.mul(re_.mul(d, og), re_.tanh_grad(tc)))
    di = re_.mul(re_.mul(dct, gg), re_.sigmoid_grad(ig))
    df = re_.mul(re_.mul(dct, cp), re_.sigmoid_grad(fg))
    dgg = re_.mul(re_.mul(dct, ig), re_.tanh_grad(gg))
    k = keep[:, t:t + 1]
    z = re_.cat([di, df, dgg, dout])
    z = re_.F(z.v * k, z.e * k)
    dz[0, :, t], dz[1, :, t] = z.v, z.e
    dh = re_.where(k, re_.chain(z, UT, bounds), d)
    dc = re_.where(k, re_.mul(dct, fg), dc)
  return {"dz": dz[0], "dh0": dh.v, "dc0": dc.v}, {"dz": dz[1], "dh0": dh.e, "dc0": dc.e}


def forward(x, W, U, bias=None, h0=None, c0=None, mask=None):
  """(seq [B, T, u], h_T [B, u], c_T [B, u], cache) for x [B, T, D]; cache is forward_gx's output."""
  x, W = np.asarray(x, np.float64), np.asarray(W, np.float64)
  b = 0.0 if bias is None else np.asarray(bias, np.float64)
  out, _ = forward_gx(x @ W + b, U, h0, c0, mask, bounds=False)
  return out["seq"], out["h_T"], out["c_T"], out


def backward(x, W, U, bias=None, h0=None, c0=None, mask=None, g_seq=None, g_h=None, g_c=None):
  """Gradients of sum(seq * g_seq) + sum(h_T * g_h) + sum(c_T * g_c): dict of dx, dW, dU, dbias ([4u], None without
  bias), dh0, dc0, and the projection's gradient dz [B, T, 4u]."""
  x, W = np.asarray(x, np.float64), np.asarray(W, np.float64)
  B, T, D = x.shape
  _, _, _, c = forward(x, W, U, bias, h0, c0, mask)
  r, _ = reverse(U, c["gates"], c["c_seq"], c0, mask, g_seq, g_h, g_c, bounds=False)
  u = c["h_prev"].shape[-1]
  z2 = r["dz"].reshape(B * T, 4 * u)
  return {"dx": (z2 @ W.T).reshape(B, T, D), "dW": x.reshape(B * T, D).T @ z2,
          "dU": c["h_prev"].reshape(B * T, u).T @ z2, "dh0": r["dh0"], "dc0": r["dc0"], "dz": r["dz"],
          "dbias": None if bias is None else z2.sum(0)}
