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
TINY = 2.0 ** -125          # one float32 denormal step, 2^-149, in units of u = 2^-24


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


def _ds(cache, dout):
  g = _f64(dout) * cache["qm"][..., None]
  dw = (g @ cache["v"].transpose(0, 2, 1)) * cache["z"]
  w = cache["w"]
  return g, dw, w * (dw - (w * dw).sum(-1, keepdims=True))


def error_bounds(cache, dout):
  """First-order bounds on the float32 kernels' absolute error, per element and in units of u = 2^-24, for out, the
  returned weights, dq, dk and dv (shapes as forward / backward return them).  They count the roundings of the kernels'
  operation order (csrc/attention.cuh, the dense modes):
    score   dot: the team's fmaf chain (ceil(dim / 8) per lane, 3 butterfly adds) times the fp32 scale; concat /
            additive: the tanh argument (two roundings: q + k, times c), tanhf (2 ulp), the chain of w_d t_d, times wc;
    weights e^{s - m} / l moves by the score's error and by l's (a sum of Tv terms), expf and __fdividef (2 ulp each),
            and the fp32 dropout factor;
    out     Tv fmafs, Tv rescales and the division by l;
    dv      Tq fmafs of w' dO;  dO . (z v - O) and its delta a chain of ceil(dv / 8) + 3 roundings with O's error;
    dq, dk  Tv (Tq) fmafs of ds times k / q (dot), or of ds wc c w_d (1 - t_d^2) with 1 - t^2 one fmaf on a t carrying
            its own error (concat / additive);
    and every operation whose result falls below 2^-126 errs by up to one denormal step: TINY per operation."""
  q, k, v, w, z, wd, t = (cache[n] for n in ("q", "k", "v", "w", "z", "wd", "t"))
  mode, scale, wc = cache["mode"], cache["scale"], cache["wc"]
  D, dv = q.shape[-1], v.shape[-1]
  Tq, Tv = q.shape[1], k.shape[1]
  n_k, n_v = -(-D // 8) + 3, -(-dv // 8) + 3
  aq, ak, av = np.abs(q), np.abs(k), np.abs(v)
  if mode == "dot":
    c = 1.0 if scale is None else float(scale)
    eS = (n_k + 1) * abs(c) * (aq @ ak.transpose(0, 2, 1))
  else:
    c = 1.0 if scale is None or mode == "additive" else float(scale)
    a = np.ones(D) if mode == "concat" or scale is None else np.abs(scale)
    cw = 1.0 if wc is None else abs(wc)
    arg = np.abs(c * (q[:, :, None, :] + k[:, None, :, :]))
    dt = 1.0 - t * t
    e_t = 2 * dt * arg + 2 * np.abs(t)                       # the argument's two roundings, tanhf's 2 ulp
    eS = cw * (a * (e_t + n_k * np.abs(t))).sum(-1) + cw * np.abs((a * t).sum(-1))
  eW = w * (eS + eS.max(-1, keepdims=True) + Tv + 6) + 4 * TINY
  eWd = z * (eW + w)
  g = _f64(dout) * cache["qm"][..., None]
  ag = np.abs(g)
  O = wd @ v
  eO = eWd @ av + (2 * Tv + 2) * (wd @ av + TINY)
  edv = eWd.transpose(0, 2, 1) @ ag + (Tq + 1) * (wd.transpose(0, 2, 1) @ ag + TINY)
  _, dw, ds = _ds(cache, dout)
  delta = (g * O).sum(-1, keepdims=True)
  e_dmd = ((n_v + 2) * ((ag @ av.transpose(0, 2, 1)) * z + (ag * np.abs(O)).sum(-1, keepdims=True))
           + (ag * eO).sum(-1, keepdims=True))
  eDS = eW * np.abs(dw - delta) + w * e_dmd + 2 * np.abs(ds) + 2 * TINY
  ads = np.abs(ds)
  if mode == "dot":
    edq = abs(c) * (eDS @ ak + (Tv + 2) * (ads @ ak + TINY))
    edk = abs(c) * (eDS.transpose(0, 2, 1) @ aq + (Tq + 2) * (ads.transpose(0, 2, 1) @ aq + TINY))
  else:
    f = cw * abs(c) * a
    e_dt = 2 * np.abs(t) * e_t + dt
    eG = f * (eDS[..., None] * dt + ads[..., None] * (e_dt + 4 * dt))
    aG = f * ads[..., None] * dt
    edq = eG.sum(2) + (Tv + 1) * (aG.sum(2) + TINY)
    edk = eG.sum(1) + (Tq + 1) * (aG.sum(1) + TINY)
  qm = cache["qm"][..., None]
  return dict(out=eO * qm, weights=eWd, dq=edq, dk=edk, dv=edv)


def weight_grad_magnitudes(cache, dout):
  """The weight gradients with ds_j = w_j (dw_j - delta) replaced by w_j (|dw_j| + |delta|) and every other factor by
  its magnitude: (dscale, dconcat_weight), dscale scalar or [dim] as backward returns it, None where backward's is.  A
  float32 ds errs relative to |dw_j| + |delta|, not to the difference, which cancels to exactly 0 at Tv = 1."""
  q, k, t, w = (cache[n] for n in ("q", "k", "t", "w"))
  mode, scale, wc = cache["mode"], cache["scale"], cache["wc"]
  _, dw, _ = _ds(cache, dout)
  m = w * (np.abs(dw) + np.abs((w * dw).sum(-1, keepdims=True)))
  if mode == "dot":
    return (None if scale is None else float((m * np.abs(q @ k.transpose(0, 2, 1))).sum())), None
  if mode == "additive":
    return (None if scale is None else (m[..., None] * np.abs(t)).sum((0, 1, 2))), None
  u = np.abs(q[:, :, None, :] + k[:, None, :, :])
  dsc = None if scale is None else float((m * abs(wc) * (u * (1.0 - t * t)).sum(-1)).sum())
  return dsc, float((m * np.abs(t).sum(-1)).sum())


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
