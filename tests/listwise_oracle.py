"""NumPy restatement of K13 (csrc/listwise.cu): TF-Ranking's ListMLE, pairwise hinge and softmax losses and NDCG on [B, L]
lists, with the rules of DESIGN.md §2 (A18).

* float64 losses and gradients of every mode (`listmle64`, `softmax64`, `hinge64`), the references of the exp/log paths;
* bit-exact float32 restatements of what can be bit-exact: the hinge loss, its gradient and pair counts (`hinge32`) and NDCG
  with integer labels (`ndcg32`), plus the kernel's fixed-order fold of per-list values (`fold`);
* the derived error bars of the exp/log paths (`listmle_bars`, `softmax_bars`, `within`).
An item with !(label >= 0) is padding.  s = pred * fp32(1/T)."""
from __future__ import annotations

import numpy as np

MAX_LIST = 1024
NONE, LISTMLE, HINGE, SOFTMAX = 0, 1, 2, 3
RED_NONE, RED_SUM, RED_AUTO = 0, 1, 2
F32 = np.float32
M32 = 0xFFFFFFFF


def fmix32(h):
  h = np.asarray(h, dtype=np.uint64) & M32
  h ^= h >> np.uint64(16)
  h = (h * np.uint64(0x85EBCA6B)) & M32
  h ^= h >> np.uint64(13)
  h = (h * np.uint64(0xC2B2AE35)) & M32
  h ^= h >> np.uint64(16)
  return h


def mix32(seed, call, b, i):
  """ListMLE's tie key f(f(f(f(seed) ^ call) ^ b) ^ i), f = murmur3's 32-bit finalizer; broadcasts over numpy arrays."""
  u = lambda x: np.asarray(x, dtype=np.uint64) & M32
  return fmix32(fmix32(fmix32(fmix32(u(seed)) ^ u(call)) ^ u(b)) ^ u(i)).astype(np.uint32)


def warps_per_cta(L: int) -> int:
  Lp = 1 << max(0, (int(L) - 1).bit_length())
  return int(min(8, max(1, 2048 // Lp)))


def valid(y) -> np.ndarray:
  return np.asarray(y) >= 0   # False for NaN


def scaled(pred, temperature: float = 1.0) -> np.ndarray:
  return (np.asarray(pred, dtype=F32) * F32(1.0 / float(temperature))).astype(F32)


def listmle_order(y, seed: int, call: int, b: int) -> np.ndarray:
  """The valid items of one list by label descending, ties by mix32(seed, call, b, i) ascending, then by i."""
  y = np.asarray(y, dtype=F32)
  idx = np.nonzero(valid(y))[0]
  key = mix32(seed, call, b, idx).astype(np.int64)
  return idx[np.lexsort((idx, key, -y[idx].astype(np.float64)))]


# ------------------------------------------------------------------------------------------------
# float64 references (one list; s already scaled, fp32)
# ------------------------------------------------------------------------------------------------
def listmle64(s, y, order):
  """(loss, dl/ds [L], T) in float64; T = sum_k |log S_k| + |s_pi(k) - m|, the scale of the loss bar."""
  s = np.asarray(s, dtype=np.float64)
  g = np.zeros(len(s))
  if len(order) == 0:
    return 0.0, g, 0.0
  m = s[order].max()
  e = np.exp(s[order] - m)
  S = np.cumsum(e[::-1])[::-1]
  terms = np.log(S) - (s[order] - m)
  g[order] = e * np.cumsum(1.0 / S) - 1.0
  return float(terms.sum()), g, float(np.abs(np.log(S)).sum() + np.abs(s[order] - m).sum())


def softmax64(s, y):
  """(loss, dl/ds, T): l = Y log sum exp(s - m) - sum y (s - m) over valid items; T = Y |lse| + sum y |s - m|."""
  s = np.asarray(s, dtype=np.float64); y = np.asarray(y, dtype=np.float64)
  v = valid(y)
  g = np.zeros(len(s))
  Y = y[v].sum() if v.any() else 0.0
  if not v.any() or Y == 0:
    return 0.0, g, 0.0
  m = s[v].max()
  t = s[v] - m
  lse = np.log(np.exp(t).sum())
  g[v] = Y * np.exp(t - lse) - y[v]
  return float(Y * lse - (y[v] * t).sum()), g, float(Y * abs(lse) + (y[v] * np.abs(t)).sum())


def hinge64(s, y):
  """(loss, dl/ds, #pairs) in float64."""
  s = np.asarray(s, dtype=np.float64); y = np.asarray(y, dtype=np.float64)
  v = valid(y)
  pair = v[:, None] & v[None, :] & (y[:, None] > y[None, :])
  h = 1.0 - (s[:, None] - s[None, :])
  cnt = int(pair.sum())
  if cnt == 0:
    return 0.0, np.zeros(len(s)), 0
  act = pair & (h > 0)
  g = (act.sum(0) - act.sum(1)) / cnt
  return float(np.where(pair, np.maximum(h, 0.0), 0.0).sum() / cnt), g, cnt


# ------------------------------------------------------------------------------------------------
# bit-exact float32 restatements ([B, L] arrays)
# ------------------------------------------------------------------------------------------------
def hinge32(s, y, w=None):
  """(l [B] fp32, dlds [B, L] fp32 with the weights, #pairs [B]): rows r_i = fp32 sum over j ascending, the list = fp32 sum
  of the rows over i ascending, / #pairs; dlds = fp32(w * c_k / #pairs) in fp64."""
  s = np.asarray(s, dtype=F32); y = np.asarray(y, dtype=F32)
  B, L = s.shape
  v = valid(y)
  w = np.ones(B, dtype=F32) if w is None else np.asarray(w, dtype=F32)
  r = np.zeros((B, L), dtype=F32)
  c = np.zeros((B, L), dtype=np.int64)
  cnt = np.zeros(B, dtype=np.int64)
  yy = np.where(v, y, F32(-1))
  for j in range(L):
    vj = v[:, j:j + 1]
    down = v & vj & (yy > yy[:, j:j + 1])
    h = (F32(1) - (s - s[:, j:j + 1])).astype(F32)
    r = np.where(down, (r + np.maximum(h, F32(0))).astype(F32), r)
    cnt += down.sum(1)
    c -= (down & (h > 0))
    up = v & vj & (yy[:, j:j + 1] > yy)
    hu = (F32(1) - (s[:, j:j + 1] - s)).astype(F32)
    c += (up & (hu > 0))
  tot = np.zeros(B, dtype=F32)
  for i in range(L):
    tot = np.where(v[:, i], (tot + r[:, i]).astype(F32), tot)
  l = np.where(cnt > 0, (tot / np.maximum(cnt, 1).astype(F32)).astype(F32), F32(0)).astype(F32)
  with np.errstate(invalid="ignore", divide="ignore"):
    gd = np.where(cnt[:, None] > 0, c / np.maximum(cnt, 1)[:, None].astype(np.float64), 0.0)
  dl = np.where(v, (w.astype(np.float64)[:, None] * gd).astype(F32), F32(0)).astype(F32)
  return l, dl, cnt


def discounts() -> np.ndarray:
  r = np.arange(1, MAX_LIST + 1, dtype=np.float64)
  return (1.0 / np.log2(r + 1.0)).astype(F32)


def _dcg32(gains, order, top, disc):
  d = F32(0)
  for r in range(top):
    d = F32(d + F32(gains[order[r]] * disc[r]))
  return d


def ndcg32(pred, y, topn=None):
  """(ndcg [B] fp32, idcg [B] fp32): gain exp2(y) - 1, ranks by pred descending (ties to the lower index), sequential fp32."""
  pred = np.asarray(pred, dtype=F32); y = np.asarray(y, dtype=F32)
  B, L = pred.shape
  disc = discounts()
  nd = np.zeros(B, dtype=F32); idcg_all = np.zeros(B, dtype=F32)
  for b in range(B):
    idx = np.nonzero(valid(y[b]))[0]
    n = len(idx)
    top = n if topn is None else min(int(topn), n)
    gains = np.zeros(L, dtype=F32)
    gains[idx] = (np.exp2(y[b, idx]) - F32(1)).astype(F32)
    ideal = idx[np.lexsort((idx, -y[b, idx].astype(np.float64)))]
    ranked = idx[np.lexsort((idx, -pred[b, idx].astype(np.float64)))]
    idcg = _dcg32(gains, ideal, top, disc)
    dcg = _dcg32(gains, ranked, top, disc)
    idcg_all[b] = idcg
    nd[b] = F32(dcg / idcg) if idcg > 0 else F32(0)
  return nd, idcg_all


def fold(values, L: int) -> float:
  """The kernel's fixed-order float64 sum of per-list values: per CTA of W lists in list order, then thread t of 32 W sums CTA
  records t, t + 32 W, ... ascending, then a pairwise tree over the threads."""
  v = np.asarray(values, dtype=np.float64)
  W = warps_per_cta(L)
  grid = max(1, -(-len(v) // W))
  pad = np.zeros(grid * W); pad[:len(v)] = v
  pad = pad.reshape(grid, W)
  rec = np.zeros(grid)
  for k in range(W):
    rec = rec + pad[:, k]
  nt = 32 * W
  rows = -(-grid // nt)
  rp = np.zeros(rows * nt); rp[:grid] = rec
  rp = rp.reshape(rows, nt)
  red = np.zeros(nt)
  for z in range(rows):
    red = red + rp[z]
  h = nt // 2
  while h > 0:
    red = np.concatenate([red[:h] + red[h:2 * h], red[h:]])
    h //= 2
  return float(red[0])


def ndcg_stats(nd, idcg, w, L: int):
  """[sum w ndcg, sum w'] as the kernel folds them; a list with IDCG = 0 weighs the mean w of the lists with IDCG > 0."""
  B = len(nd)
  w = np.ones(B, dtype=F32) if w is None else np.asarray(w, dtype=F32)
  pos = idcg > 0
  wd = w.astype(np.float64)
  t1 = fold(np.where(pos, wd * nd.astype(np.float64), 0.0), L)
  t2 = fold(np.where(pos, wd, 0.0), L)
  t3 = fold(pos.astype(np.float64), L)
  t4 = fold((~pos).astype(np.float64), L)
  return np.array([t1, t2 + t4 * (t2 / t3 if t3 > 0 else 0.0)])


def reduce_loss(per_list32, B: int, L: int, reduction: int):
  """The fp32 loss scalar from the fp32 weighted per-list losses."""
  t = fold(np.asarray(per_list32, dtype=F32).astype(np.float64), L)
  return F32(t / B if (reduction == RED_AUTO and B > 0) else t)


# ------------------------------------------------------------------------------------------------
# whole calls
# ------------------------------------------------------------------------------------------------
def forward64(mode, pred, y, w=None, temperature=1.0, seed=0, call=0):
  """(l [B] float64 unweighted, dl/ds [B, L] float64 unweighted, scale T [B], n [B])."""
  s = scaled(pred, temperature)
  y = np.asarray(y, dtype=F32)
  B, L = s.shape
  l = np.zeros(B); g = np.zeros((B, L)); T = np.zeros(B); n = valid(y).sum(1)
  for b in range(B):
    if mode == LISTMLE:
      l[b], g[b], T[b] = listmle64(s[b], y[b], listmle_order(y[b], seed, call, b))
    elif mode == SOFTMAX:
      l[b], g[b], T[b] = softmax64(s[b], y[b])
    elif mode == HINGE:
      l[b], g[b], _ = hinge64(s[b], y[b])
  return l, g, T, n


def backward32(dlds, g, reduction: int, temperature=1.0):
  """dx = (c * dlds) * fp32(1/T) + 0, c = g[b] (NONE), g (SUM), g / B (AUTO) in fp32; the + 0 makes a zero gradient +0."""
  dlds = np.asarray(dlds, dtype=F32)
  B = dlds.shape[0]
  g = np.asarray(g, dtype=F32).reshape(-1)
  c = g[:, None] if reduction == RED_NONE else (F32(g[0] / F32(B)) if reduction == RED_AUTO else g[0])
  return (((c * dlds).astype(F32) * F32(1.0 / float(temperature))).astype(F32) + F32(0)).astype(F32)


# ------------------------------------------------------------------------------------------------
# error bars of the exp/log paths (ListMLE, softmax)
# ------------------------------------------------------------------------------------------------
# The kernel computes these modes in float64 (exp, log, sums over n <= 1024 items) and rounds once to fp32; the oracle is
# float64 too.  Each side's float64 error is at most ~4 n ulp(2^-53) of the summed magnitudes; 2^-40 n T leaves a 2^7 margin.
# The fp32 results carry two roundings (the list loss, then w * l; the gradient once): 2^-22 relative covers them.
LOSS_REL, GRAD_REL, F64_SLACK = 2.0 ** -22, 2.0 ** -23, 2.0 ** -40


def listmle_bars(l, g, T, n, w=None):
  """(per-list bar [B] of w l, per-item bar [B, L] of w dl/ds) for ListMLE: dl/ds_k = e_k P_k - 1, so its magnitude scale is
  |g| + 1 per item."""
  w = np.ones(len(l)) if w is None else np.abs(np.asarray(w, dtype=np.float64))
  lb = w * (LOSS_REL * np.abs(l) + F64_SLACK * n * T)
  gb = w[:, None] * (GRAD_REL * np.abs(g) + F64_SLACK * n[:, None] * (np.abs(g) + 1.0))
  return lb, gb


def softmax_bars(l, g, T, n, y, w=None):
  """The same bars for softmax: dl/ds_i = Y p_i - y_i, magnitude scale Y p_i + y_i <= |g| + 2 y_i."""
  w = np.ones(len(l)) if w is None else np.abs(np.asarray(w, dtype=np.float64))
  yv = np.where(valid(y), np.asarray(y, dtype=np.float64), 0.0)
  lb = w * (LOSS_REL * np.abs(l) + F64_SLACK * n * T)
  gb = w[:, None] * (GRAD_REL * np.abs(g) + F64_SLACK * n[:, None] * (np.abs(g) + 2.0 * yv + 2.0 ** -30))
  return lb, gb


def within(got, ref, bar) -> bool:
  got = np.asarray(got, dtype=np.float64); ref = np.asarray(ref, dtype=np.float64)
  return bool(np.all(np.abs(got - ref) <= bar))
