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
    a = _aug_argmax(xt, cent)
    for l in range(L):
      m = np.nonzero(a == l)[0]
      if m.size:
        cent[l] = _ordered_mean(xt[m])
  leaf = _aug_argmax(x, cent)
  order = np.argsort(leaf, kind="stable").astype(np.int32)
  offsets = np.concatenate([[0], np.cumsum(np.bincount(leaf, minlength=L))]).astype(np.int32)
  rt = xt - cent[_aug_argmax(xt, cent)]
  cb = np.zeros((B, 16, dpb), F32)
  init = rt[np.searchsorted(train_rows, perm[np.arange(16) % n_train])]
  for b, (c0, w) in enumerate(_blocks(d, dpb)):
    cb[b, :, :w] = init[:, c0:c0 + w]
  for _ in range(CODEBOOK_ITERATIONS):
    codes = _encode(rt, cb, dpb)
    for b, (c0, w) in enumerate(_blocks(d, dpb)):
      for j in range(16):
        m = np.nonzero(codes[:, b] == j)[0]
        if m.size:
          cb[b, j, :w] = _ordered_mean(rt[m, c0:c0 + w])
  codes = _encode((x - cent[leaf])[order], cb, dpb)
  return {"centroids": cent, "leaf_offsets": offsets, "order": order, "codebooks": cb, "codes": pack(codes),
          "perm": perm, "train_rows": train_rows, "leaf": leaf}


def lut(q: np.ndarray, cb: np.ndarray, dpb: int):
  """(T8 int [Q, B, 16], s float32 [Q]) of DESIGN.md §2."""
  q = np.ascontiguousarray(q, F32)
  T = np.stack([orc.scores(np.ascontiguousarray(q[:, c0:c0 + w]), np.ascontiguousarray(cb[b, :, :w]))
                for b, (c0, w) in enumerate(_blocks(q.shape[1], dpb))], 1)
  m = np.abs(T).max(axis=(1, 2))
  s = np.where(m > 0, m / F32(127.0), F32(0)).astype(F32)
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
