"""Float64 NumPy oracle of tf-keras 2.x's BaseDenseAttention (layers.Attention, layers.AdditiveAttention), forward and
backward, for the three score modes, with masks and a given dropout keep mask.  DESIGN.md §2 (A27) restates it:

  scores   "dot":      s = (q . k) * scale                          (scale a scalar, or none)
           "concat":   s = wc * sum_d tanh(scale * (q_d + k_d))     (scale a scalar, or none; wc concat_score_weight)
           "additive": s = sum_d scale_d * tanh(q_d + k_d)          (scale [dim], or none)
  mask     keep(b, i, j) = value_mask[b, j] & (j <= i if causal); a dropped score gets s -= 1e9 in fp32;
           w = softmax_j(s)
  dropout  w' = keep_drop ? w / (1 - rate) : 0 (keep_drop = regularization_oracle.dropout_keep((B, Tq, Tv), rate, seed,
           call) in training, all kept otherwise)
  output   out[b, i] = query_mask[b, i] * sum_j w'_ij v_j;  the returned weights are w'."""
from __future__ import annotations

import numpy as np

MODES = ("dot", "concat", "additive")


def _f64(a):
  return None if a is None else np.asarray(a, dtype=np.float64)


def keep_mask(B, Tq, Tv, value_mask=None, causal=False) -> np.ndarray:
  """bool [B, Tq, Tv]: the scores the softmax keeps."""
  keep = np.ones((B, Tq, Tv), bool)
  if value_mask is not None:
    keep &= np.asarray(value_mask).astype(bool)[:, None, :]
  if causal:
    keep &= np.tril(np.ones((Tq, Tv), bool))[None]
  return keep


def _scores(q, k, mode, scale, wc):
  if mode == "dot":
    s = q @ k.transpose(0, 2, 1)
    return (s if scale is None else s * scale), None
  u = q[:, :, None, :] + k[:, None, :, :]
  if mode == "concat":
    t = np.tanh(u if scale is None else scale * u)
    return wc * t.sum(-1), t
  t = np.tanh(u)
  return (t.sum(-1) if scale is None else (t * scale).sum(-1)), t


def forward(q, k, v, mode="dot", scale=None, concat_weight=None, query_mask=None, value_mask=None, causal=False,
            drop_keep=None, rate=0.0):
  """(out [B, Tq, dv], weights w' [B, Tq, Tv], cache for backward)."""
  q, k, v = _f64(q), _f64(k), _f64(v)
  scale = None if scale is None else np.asarray(scale, np.float64).reshape(-1 if mode == "additive" else ())
  wc = None if concat_weight is None else float(np.asarray(concat_weight).reshape(()))
  B, Tq, _ = q.shape
  Tv = k.shape[1]
  s, t = _scores(q, k, mode, scale, wc)
  keep = keep_mask(B, Tq, Tv, value_mask, causal)
  s = np.where(keep, s, (s - 1e9).astype(np.float32).astype(np.float64))   # fp32: a fully masked row is uniform
  e = np.exp(s - s.max(-1, keepdims=True))
  w = e / e.sum(-1, keepdims=True)
  z = np.ones_like(w) if drop_keep is None else np.where(drop_keep, 1.0 / (1.0 - rate), 0.0)
  wd = w * z
  out = wd @ v
  qm = np.ones((B, Tq)) if query_mask is None else np.asarray(query_mask).astype(bool).astype(np.float64)
  out = out * qm[..., None]
  cache = dict(q=q, k=k, v=v, mode=mode, scale=scale, wc=wc, t=t, w=w, z=z, wd=wd, qm=qm)
  return out, wd, cache


def backward(cache, dout):
  """(dq, dk, dv, dscale, dconcat_weight): dscale has scale's shape (None without a scale), dconcat_weight is a float
  (None outside "concat").  With key = value the caller adds dk to dv."""
  q, k, v, w, z, wd, t = (cache[n] for n in ("q", "k", "v", "w", "z", "wd", "t"))
  mode, scale, wc = cache["mode"], cache["scale"], cache["wc"]
  g = _f64(dout) * cache["qm"][..., None]
  dv = wd.transpose(0, 2, 1) @ g
  dw = (g @ v.transpose(0, 2, 1)) * z
  ds = w * (dw - (w * dw).sum(-1, keepdims=True))
  dscale = dwc = None
  if mode == "dot":
    c = 1.0 if scale is None else float(scale)
    dq = c * ds @ k
    dk = c * ds.transpose(0, 2, 1) @ q
    if scale is not None:
      dscale = np.float64((ds * (q @ k.transpose(0, 2, 1))).sum())
    return dq, dk, dv, dscale, dwc
  dt = 1.0 - t * t
  if mode == "concat":
    c = 1.0 if scale is None else float(scale)
    G = ds[..., None] * wc * c * dt
    u = q[:, :, None, :] + k[:, None, :, :]
    if scale is not None:
      dscale = np.float64((ds * wc * (u * dt).sum(-1)).sum())
    dwc = float((ds * t.sum(-1)).sum())
  else:
    a = np.ones(q.shape[-1]) if scale is None else scale
    G = ds[..., None] * a * dt
    if scale is not None:
      dscale = (ds[..., None] * t).sum((0, 1, 2))
  return G.sum(2), G.sum(1), dv, dscale, dwc


def weight_grad_rows(cache, dout):
  """The per-query-row contributions [B, Tq] to the scalar weight gradients (dscale of "dot" / "concat", and
  dconcat_weight), whose sums backward() returns: (dscale rows or None, dconcat_weight rows or None)."""
  q, k, v, w, z, t = (cache[n] for n in ("q", "k", "v", "w", "z", "t"))
  mode, scale, wc = cache["mode"], cache["scale"], cache["wc"]
  g = _f64(dout) * cache["qm"][..., None]
  dw = (g @ v.transpose(0, 2, 1)) * z
  ds = w * (dw - (w * dw).sum(-1, keepdims=True))
  if mode == "dot":
    return (None if scale is None else (ds * (q @ k.transpose(0, 2, 1))).sum(-1)), None
  if mode != "concat":
    return None, None
  u = q[:, :, None, :] + k[:, None, :, :]
  rows = None if scale is None else (ds * wc * (u * (1.0 - t * t)).sum(-1)).sum(-1)
  return rows, (ds * t.sum(-1)).sum(-1)
