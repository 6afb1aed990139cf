"""float64 NumPy restatement of tf.keras.layers.MultiHeadAttention (attention over the sequence axis, no dropout) and of
tf.keras.layers.LayerNormalization (last axis), forward and backward: the reference the K21 / K22 tests compare against.

MultiHeadAttention follows Keras's order: the projections (EinsumDense with the kernels viewed as 2-D), the query times
float32(1 / sqrt(dk)), the scores, the combined mask applied as tf-keras's Softmax does (a dropped score becomes
float32(s + (-1e9)), so a fully masked row is uniform), the softmax over S, P.V and the output projection.  The backward
treats the mask adder as an addition (derivative 1), as autograd does."""
import numpy as np

MASK_ADDER = -1e9
TINY = 2.0 ** -125          # one float32 denormal step, 2^-149, in units of u = 2^-24


def _f64(a):
  return None if a is None else np.asarray(a, np.float64)


def combined_mask(B, T, S, query_mask=None, value_mask=None, key_mask=None, attention_mask=None, causal=False):
  """keep [B, T, S] bool (tf-keras _compute_attention_mask), or None when no mask is given."""
  keep = None

  def both(a, b):
    return b if a is None else a & b

  if query_mask is not None:
    keep = both(keep, (np.asarray(query_mask) != 0)[:, :, None])
  if value_mask is not None:
    keep = both(keep, (np.asarray(value_mask) != 0)[:, None, :])
  if key_mask is not None:
    keep = both(keep, (np.asarray(key_mask) != 0)[:, None, :])
  if causal:
    keep = both(keep, np.tril(np.ones((T, S), bool))[None])
  if attention_mask is not None:
    keep = both(keep, np.asarray(attention_mask) != 0)
  return None if keep is None else np.broadcast_to(keep, (B, T, S))


def scale_of(dk):
  return float(np.float32(1.0 / np.sqrt(float(dk))))


def core_forward(Q, K, V, keep):
  """Q [B, T, H, dk], K [B, S, H, dk], V [B, S, H, dv] (float64; Q not yet scaled) -> (O [B, T, H, dv], P [B, H, T,
  S], Qs)."""
  Qs = Q * scale_of(Q.shape[-1])
  s = np.einsum("bthd,bshd->bhts", Qs, K)
  if keep is not None:
    k = np.broadcast_to(keep[:, None], s.shape)
    s = np.where(k, s, (s + MASK_ADDER).astype(np.float32).astype(np.float64))
  e = np.exp(s - s.max(-1, keepdims=True))
  P = e / e.sum(-1, keepdims=True)
  return np.einsum("bhts,bshd->bthd", P, V), P, Qs


def core_backward(Q, K, V, P, Qs, dO):
  """(dQ, dK, dV) of the core from dO [B, T, H, dv]."""
  dP = np.einsum("bthd,bshd->bhts", dO, V)
  dV = np.einsum("bhts,bthd->bshd", P, dO)
  dS = P * (dP - (dP * P).sum(-1, keepdims=True))
  dQ = np.einsum("bhts,bshd->bthd", dS, K) * scale_of(Q.shape[-1])
  dK = np.einsum("bhts,bthd->bshd", dS, Qs)
  return dQ, dK, dV


def core_error_bounds(Q, K, V, P, Qs, dO):
  """First-order bounds on the float32 kernels' absolute error, per element and in units of u = 2^-24, for O, P, dQ,
  dK and dV of the core (shapes as core_forward / core_backward return them).  They count the roundings of the
  kernels' operation order (csrc/attention.cuh):
    score   the team's fmaf chain of ceil(dk / 8) terms per lane, 3 butterfly adds and the fp32 q * 1/sqrt(dk): n_k
            roundings of magnitude A = sum_d |qs_d k_d|;
    P       e^{s - m} / l moves by the score's error, by l's (a sum of S terms, at most the largest score error plus S
            roundings), and by expf and __fdividef (2 ulp each);
    O       S fmafs into o, S rescales by e^{m_old - m}, the division by l;
    dV      T fmafs of p dO;  dP = dO . v and delta = dO . O are chains of n_v roundings;
    dK, dQ  T (S) fmafs of ds q (ds k) over the staged q * 1/sqrt(dk) (k), ds = p (dP - delta) with both errors;
    and every operation whose result falls below 2^-126 (a p of e^-100, its products) errs by up to one denormal
    step, 2^-149 absolute: TINY in units of u, once per operation of the chain."""
  dk, dv = Q.shape[-1], V.shape[-1]
  S, T = K.shape[1], Q.shape[1]
  n_k, n_v = -(-dk // 8) + 4, -(-dv // 8) + 3
  aQs, aK, aV, adO = np.abs(Qs), np.abs(K), np.abs(V), np.abs(dO)
  eS = n_k * np.einsum("bthd,bshd->bhts", aQs, aK)
  eP = P * (eS + eS.max(-1, keepdims=True) + S + 6) + 4 * TINY
  PaV = np.einsum("bhts,bshd->bthd", P, aV)
  eO = np.einsum("bhts,bshd->bthd", eP, aV) + (2 * S + 2) * PaV + (2 * S + 2) * TINY
  eV = np.einsum("bhts,bthd->bshd", eP, adO) + (T + 1) * np.einsum("bhts,bthd->bshd", P, adO) + (T + 1) * TINY
  O = np.einsum("bhts,bshd->bthd", P, V)
  dP = np.einsum("bthd,bshd->bhts", dO, V)
  delta = np.einsum("bthd,bthd->bht", dO, O)[..., None]
  e_delta = (n_v * np.einsum("bthd,bthd->bht", adO, np.abs(O)) + np.einsum("bthd,bthd->bht", adO, eO))[..., None]
  e_dP = n_v * np.einsum("bthd,bshd->bhts", adO, aV)
  dS = P * (dP - delta)
  eDS = eP * np.abs(dP - delta) + P * (e_dP + e_delta) + 2 * np.abs(dS) + 2 * TINY
  aDS = np.abs(dS)
  eK = np.einsum("bhts,bthd->bshd", eDS, aQs) + (T + 2) * (np.einsum("bhts,bthd->bshd", aDS, aQs) + TINY)
  eQ = scale_of(dk) * (np.einsum("bhts,bshd->bthd", eDS, aK) + (S + 2) * (np.einsum("bhts,bshd->bthd", aDS, aK) + TINY))
  return dict(O=eO, P=eP, dQ=eQ, dK=eK, dV=eV)


def _proj(x, W, b):
  y = x @ W.reshape(W.shape[0], -1)
  return y if b is None else y + b.reshape(-1)


def mha_forward(query, value, key, Wq, Wk, Wv, Wo, bq=None, bk=None, bv=None, bo=None, keep=None):
  """(out [B, T, D_out], P [B, H, T, S], cache).  key None = value.  keep from combined_mask."""
  query, value = _f64(query), _f64(value)
  key = value if key is None else _f64(key)
  Wq, Wk, Wv, Wo, bq, bk, bv, bo = (_f64(a) for a in (Wq, Wk, Wv, Wo, bq, bk, bv, bo))
  B, T, _ = query.shape
  S = value.shape[1]
  H, dk, dv = Wq.shape[1], Wq.shape[2], Wv.shape[2]
  Q = _proj(query, Wq, bq).reshape(B, T, H, dk)
  K = _proj(key, Wk, bk).reshape(B, S, H, dk)
  V = _proj(value, Wv, bv).reshape(B, S, H, dv)
  O, P, Qs = core_forward(Q, K, V, keep)
  Of = O.reshape(B, T, H * dv)
  out = Of @ Wo.reshape(H * dv, -1)
  if bo is not None:
    out = out + bo
  return out, P, dict(query=query, value=value, key=key, Q=Q, K=K, V=V, P=P, Qs=Qs, Of=Of, W=(Wq, Wk, Wv, Wo))


def mha_backward(cache, g, key_is_value=False):
  """Every gradient from g [B, T, D_out]: dquery, dvalue, dkey (None when key_is_value: folded into dvalue), dWq, dWk,
  dWv, dWo, dbq, dbk, dbv, dbo (weights in Keras's shapes)."""
  g = _f64(g)
  Wq, Wk, Wv, Wo = cache["W"]
  Q, K, V, P, Qs, Of = (cache[k] for k in ("Q", "K", "V", "P", "Qs", "Of"))
  B, T, H, dk = Q.shape
  S, dv = V.shape[1], V.shape[3]
  Wo2 = Wo.reshape(H * dv, -1)
  r = {"dWo": np.einsum("btj,bto->jo", Of, g).reshape(Wo.shape), "dbo": g.sum((0, 1))}
  dO = (g @ Wo2.T).reshape(B, T, H, dv)
  dQ, dK, dV = core_backward(Q, K, V, P, Qs, dO)
  for name, x, W, d in (("q", cache["query"], Wq, dQ), ("k", cache["key"], Wk, dK), ("v", cache["value"], Wv, dV)):
    d2 = d.reshape(d.shape[0], d.shape[1], -1)
    W2 = W.reshape(W.shape[0], -1)
    r["d" + {"q": "query", "k": "key", "v": "value"}[name]] = d2 @ W2.T
    r["dW" + name] = np.einsum("bti,btj->ij", x, d2).reshape(W.shape)
    r["db" + name] = d2.sum((0, 1)).reshape(W.shape[1:])
  # dbk = sum_{b,s} dK is exactly zero (a per-head shift of every key moves a row's scores alike, and the softmax ignores
  # it): what a float32 computation leaves is the cancellation of these magnitudes
  r["dbk_terms"] = np.abs(dK).sum((0, 1))
  if key_is_value:
    r["dvalue"] = r["dvalue"] + r["dkey"]
    r["dkey"] = None
  return r


def layer_norm_forward(x, gamma=None, beta=None, eps=1e-3):
  """(y, mean, rstd) over the last axis, population variance."""
  x = _f64(x)
  mu = x.mean(-1, keepdims=True)
  var = ((x - mu) ** 2).mean(-1, keepdims=True)
  rs = 1.0 / np.sqrt(var + eps)
  y = (x - mu) * rs
  if gamma is not None:
    y = y * _f64(gamma)
  if beta is not None:
    y = y + _f64(beta)
  return y, mu[..., 0], rs[..., 0]


def layer_norm_backward(x, gamma, g, eps=1e-3):
  """(dx, dgamma, dbeta) from g = dL/dy."""
  x, g = _f64(x), _f64(g)
  d = x.shape[-1]
  _, mu, rs = layer_norm_forward(x, None, None, eps)
  xh = (x - mu[..., None]) * rs[..., None]
  gg = g if gamma is None else g * _f64(gamma)
  dx = rs[..., None] * (gg - gg.mean(-1, keepdims=True) - xh * (gg * xh).sum(-1, keepdims=True) / d)
  lead = tuple(range(x.ndim - 1))
  return dx, (g * xh).sum(lead), g.sum(lead)
