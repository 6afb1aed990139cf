"""NumPy restatement of the tree-AH rules of DESIGN.md §2 (TreeAH, K9) -- the bar the GPU index and search meet bit for bit.

Canonical dots and selections come from oracle/oracle.py (`scores`: the sequential fmaf chain from +0.0f; `topk_scan`:
(score desc, index asc)).  Float64 sums are sequential (`np.cumsum(...)[-1]`, not the pairwise `np.sum`); every other
step is one NumPy float32 operation, i.e. one correctly rounded IEEE operation."""
from __future__ import annotations

import numpy as np

from oracle import oracle as orc

MAX_TRAIN = 100000
CODEBOOK_ITERATIONS = 10
F32 = np.float32
SEARCH_BUDGET = 512 << 20     # bytes of per-chunk search lists (TA_SEARCH_BUDGET)
MERGE_MAX_LISTS = 64          # the sorted-list tree merge's limits (tfrs_topk_merge_sorted_strided)
MERGE_MAX_SMEM = 160 * 1024


def _norms(c: np.ndarray) -> np.ndarray:
  """Canonical dot of every row with itself."""
  return np.array([orc.scores(c[i:i + 1], c[i:i + 1])[0, 0] for i in range(c.shape[0])], F32)


def _aug_argmax(y: np.ndarray, c: np.ndarray) -> np.ndarray:
  """Top-1 of [y, 1] . [c, -0.5f |c|^2] (squared L2), ties to the lower center."""
  ay = np.concatenate([y, np.ones((y.shape[0], 1), F32)], 1)
  ac = np.concatenate([c, (F32(-0.5) * _norms(c))[:, None]], 1)
  return orc.topk_scan(ay, ac, 1)[1][:, 0]


def _ordered_mean(rows: np.ndarray) -> np.ndarray:
  return (np.cumsum(rows.astype(np.float64), axis=0)[-1] / rows.shape[0]).astype(F32)


def _blocks(d: int, dpb: int):
  return [(b * dpb, min(dpb, d - b * dpb)) for b in range(-(-d // dpb))]


def _encode(r: np.ndarray, cb: np.ndarray, dpb: int) -> np.ndarray:
  """[n, B] codes of residuals r: per block the nearest of the 16 centers (augmented dot over the block's dims + 1)."""
  out = np.empty((r.shape[0], cb.shape[0]), np.int64)
  for b, (c0, w) in enumerate(_blocks(r.shape[1], dpb)):
    out[:, b] = _aug_argmax(np.ascontiguousarray(r[:, c0:c0 + w]), np.ascontiguousarray(cb[b, :, :w]))
  return out


def update_centroids(xt: np.ndarray, a: np.ndarray, cent: np.ndarray) -> np.ndarray:
  """One Lloyd step: every leaf with members becomes their ordered mean; an empty leaf keeps its centroid."""
  cent = cent.copy()
  for l in range(cent.shape[0]):
    m = np.nonzero(a == l)[0]
    if m.size:
      cent[l] = _ordered_mean(xt[m])
  return cent


def update_codebooks(rt: np.ndarray, codes: np.ndarray, cb: np.ndarray, dpb: int) -> np.ndarray:
  """One codebook step: center j of block b becomes the ordered mean of the residual blocks coded j; a center without
  members keeps its value, and the last block's unused dims are left as they are."""
  cb = cb.copy()
  for b, (c0, w) in enumerate(_blocks(rt.shape[1], dpb)):
    for j in range(16):
      m = np.nonzero(codes[:, b] == j)[0]
      if m.size:
        cb[b, j, :w] = _ordered_mean(rt[m, c0:c0 + w])
  return cb


def pack(codes: np.ndarray) -> np.ndarray:
  """[n, B] codes -> int32 words [n, ceil(B/8)]: block 8w + e in bits 4e..4e+3."""
  n, B = codes.shape
  W = (B + 7) // 8
  full = np.zeros((n, W * 8), np.uint64)
  full[:, :B] = codes
  words = np.zeros((n, W), np.uint64)
  for e in range(8):
    words |= full[:, e::8] << np.uint64(4 * e)
  return words.astype(np.uint32).view(np.int32)


def unpack(words: np.ndarray, B: int) -> np.ndarray:
  w = words.view(np.uint32).astype(np.int64)
  return np.stack([(w[:, b // 8] >> (4 * (b % 8))) & 15 for b in range(B)], 1)


def build(x, num_leaves: int, training_iterations: int, dpb: int) -> dict:
  """The index of DESIGN.md §2, with the same tensors as ops.tree_ah_build (plus `perm` and `train_rows`)."""
  x = np.ascontiguousarray(x, F32)
  N, d = x.shape
  n_train = min(N, MAX_TRAIN)
  L = min(num_leaves, n_train)
  B = -(-d // dpb)
  perm = np.random.default_rng(0).permutation(N)
  train_rows = np.sort(perm[:n_train])
  xt = x[train_rows]
  cent = x[perm[:L]].copy()
  for _ in range(training_iterations):
    cent = update_centroids(xt, _aug_argmax(xt, cent), cent)
  leaf = _aug_argmax(x, cent)
  order = np.argsort(leaf, kind="stable").astype(np.int32)
  offsets = np.concatenate([[0], np.cumsum(np.bincount(leaf, minlength=L))]).astype(np.int32)
  rt = xt - cent[_aug_argmax(xt, cent)]
  cb = np.zeros((B, 16, dpb), F32)
  init = rt[np.searchsorted(train_rows, perm[np.arange(16) % n_train])]
  for b, (c0, w) in enumerate(_blocks(d, dpb)):
    cb[b, :, :w] = init[:, c0:c0 + w]
  for _ in range(CODEBOOK_ITERATIONS):
    cb = update_codebooks(rt, _encode(rt, cb, dpb), cb, dpb)
  codes = _encode((x - cent[leaf])[order], cb, dpb)
  return {"centroids": cent, "leaf_offsets": offsets, "order": order, "codebooks": cb, "codes": pack(codes),
          "perm": perm, "train_rows": train_rows, "leaf": leaf}


def table(q: np.ndarray, cb: np.ndarray, dpb: int):
  """(T float32 [Q, B, 16], s float32 [Q]): the canonical dots of every query block with every center, and the scale."""
  q = np.ascontiguousarray(q, F32)
  T = np.stack([orc.scores(np.ascontiguousarray(q[:, c0:c0 + w]), np.ascontiguousarray(cb[b, :, :w]))
                for b, (c0, w) in enumerate(_blocks(q.shape[1], dpb))], 1)
  m = np.abs(T).max(axis=(1, 2))
  return T, np.where(m > 0, m / F32(127.0), F32(0)).astype(F32)


def lut(q: np.ndarray, cb: np.ndarray, dpb: int):
  """(T8 int [Q, B, 16], s float32 [Q]) of DESIGN.md §2."""
  T, s = table(q, cb, dpb)
  safe = np.where(s > 0, s, F32(1))[:, None, None]
  T8 = np.where(s[:, None, None] > 0, np.rint(T / safe), 0).astype(np.int64)
  return T8, s


def search(index: dict, x, q, k: int, num_leaves_to_search: int, dpb: int, num_reordering_candidates=None):
  """(scores [Q, k] float32, row ids [Q, k] int64) with (NaN, 0) padding."""
  q = np.ascontiguousarray(q, F32)
  x = np.ascontiguousarray(x, F32)
  cent, off, order = index["centroids"], index["leaf_offsets"], index["order"]
  L = cent.shape[0]
  B = index["codebooks"].shape[0]
  P = min(num_leaves_to_search, L)
  k_pre = max(num_reordering_candidates or k, k)
  ps, pl = orc.topk_scan(q, cent, P)
  T8, s = lut(q, index["codebooks"], dpb)
  codes = unpack(index["codes"], B)
  out_s = np.full((q.shape[0], k), np.nan, F32)
  out_i = np.zeros((q.shape[0], k), np.int64)
  for i in range(q.shape[0]):
    pos = np.concatenate([np.arange(off[l], off[l + 1]) for l in pl[i]])
    dots = np.concatenate([np.full(off[l + 1] - off[l], ps[i, p], F32) for p, l in enumerate(pl[i])])
    isum = T8[i][np.arange(B)[None, :], codes[pos]].sum(1)
    a = (dots + s[i] * isum.astype(F32)).astype(F32)
    rows = order[pos].astype(np.int64)
    sel = np.lexsort((rows, -a))[:k_pre]
    rows, a = rows[sel], a[sel]
    if num_reordering_candidates is not None and rows.size:
      a = orc.scores(q[i:i + 1], x[rows])[0]
      sel = np.lexsort((rows, -a))
      rows, a = rows[sel], a[sel]
    n = min(k, rows.size)
    out_s[i, :n] = a[:n]
    out_i[i, :n] = rows[:n]
  return out_s, out_i


# ---- the search plan, restated so that tests can aim at its edges ------------------------------------------------------
def slices(Q: int, P: int, N: int, L: int, sms: int) -> int:
  """Slices per (query, probed leaf): enough CTAs for two waves of `sms` SMs, never fewer than 256 rows per slice of an
  average leaf, 1..64."""
  want = -(-2 * sms // (Q * P))
  return max(1, min(64, want, (N // L) // 256))


def query_chunk(Q: int, P: int, S: int, B: int, k: int, kp: int, reorder: bool) -> int:
  """Queries per chunk: the Q x P x S lists of k' entries (and the rest of a query's workspace) within SEARCH_BUDGET."""
  W = (B + 7) // 8
  per_q = P * S * kp * 12 + kp * 12 + W * 128 + 4 + P * 12 + (k * 12 if reorder else 0) + P * 24
  return max(1, min(Q, SEARCH_BUDGET // per_q))


def merge_region(n_lists: int, k_in: int, k_out: int) -> int:
  """Entries of the largest level of the sorted-list merge tree."""
  ko = min(k_out, n_lists * k_in)
  region, n, c = n_lists * k_in, n_lists, k_in
  while n > 2:
    n, c = (n + 1) // 2, min(2 * c, ko)
    region = max(region, n * c)
  return region


def tree_merge(n_lists: int, k_in: int, k_out: int) -> bool:
  """True when the P x S lists merge in the shared-memory tree, False when they take the sorting merge."""
  return n_lists <= MERGE_MAX_LISTS and merge_region(n_lists, k_in, k_out) * 24 <= MERGE_MAX_SMEM and k_out <= 2048


def _factor(c, t):
  """A float32 v with fl(v * c) == t exactly (searched around t / c), or None."""
  c, t = F32(c), F32(t)
  if c == 0:
    return None
  up = down = F32(t / c)
  for _ in range(32):
    for v in (up, down):
      if F32(v * c) == t:
        return v
    up, down = np.nextafter(up, F32(np.inf)), np.nextafter(down, F32(-np.inf))
  return None


def half_tie_query(cb: np.ndarray, d: int, dpb: int, t: float):
  """A query whose table (`table`) has max |T| = 127, so s = 1, and holds the half-integer t exactly: the first dim of
  one block scales that block's largest center to 127, the first dim of another block scales its largest center to t,
  every other dim is 0.  The LUT entry is then rint(t), which `__float2int_rn` must round half to even.  None when d has
  a single block or no pair of blocks has float32 factors that hit both targets exactly."""
  top = [int(np.abs(cb[b, :, 0]).argmax()) for b in range(cb.shape[0])]
  for b0 in range(cb.shape[0]):
    v = _factor(cb[b0, top[b0], 0], 127.0)
    for b1 in range(cb.shape[0]):
      w = None if b1 == b0 or v is None else _factor(cb[b1, top[b1], 0], t)
      if w is not None:
        q = np.zeros(d, F32)
        q[b0 * dpb], q[b1 * dpb] = v, w
        return q
  return None
