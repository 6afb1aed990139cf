"""Oracle of the text and numeric feature rules (DESIGN.md §2, A21): TextVectorization, Discretization, Normalization and
GlobalAveragePooling1D restated with Python `bytes` operations and NumPy float32, one IEEE operation at a time.  Test
infrastructure: the product never imports it.

The rules are recalled from tf-keras / TF sources; there is no in-tree copy, so they are unpinned against Keras.  The
tf-keras docstring known answers (KNOWN_*) pin what they can."""
from __future__ import annotations

import os
import re
import string
from typing import Dict, List, Optional, Sequence

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

PUNCTUATION = string.punctuation.encode("ascii")          # Keras DEFAULT_STRIP_REGEX deletes exactly these 32 bytes
WHITESPACE = b" \t\n\x0b\x0c\r"                           # absl ascii_isspace
_SPLIT = re.compile(b"[" + re.escape(WHITESPACE) + b"]+")
_UPPER = bytes(range(ord("A"), ord("Z") + 1))
_LOWER_TABLE = bytes.maketrans(_UPPER, _UPPER.lower())
EPSILON = np.float32(1e-7)

# tf-keras docstring known answers
KNOWN_ADAPT = dict(adapt=["foo", "bar", "baz"], max_tokens=5000, output_sequence_length=4,
                   inputs=[["foo qux bar"], ["qux baz"]], expected=[[2, 1, 4, 0], [1, 3, 0, 0]])
KNOWN_VOCAB = dict(vocabulary=["earth", "wind", "and", "fire"], inputs=[["earth wind and fire"], ["fire and earth michigan"]],
                   expected=[[2, 3, 4, 5], [5, 4, 2, 1]])
KNOWN_NORMALIZATION = dict(adapt=[1.0, 2.0, 3.0, 4.0, 5.0], inputs=[1.0, 2.0, 3.0], mean=3.0, variance=2.0,
                           expected=[-1.4142135, -0.70710677, 0.0])


def as_bytes(s) -> bytes:
  return s.encode("utf-8") if isinstance(s, str) else bytes(s)


# ---- text ------------------------------------------------------------------------------------------------------------
def standardize(s: bytes, lower: bool = True, strip: bool = True) -> bytes:
  if lower:
    s = s.translate(_LOWER_TABLE)                        # ASCII only: bytes >= 0x80 stay as they are
  if strip:
    s = s.translate(None, PUNCTUATION)
  return s


def split(s: bytes) -> List[bytes]:
  return [t for t in _SPLIT.split(s) if t]


def tokens(s, lower: bool = True, strip: bool = True) -> List[bytes]:
  return split(standardize(as_bytes(s), lower, strip))


def vectorize(strings: Sequence, vocabulary: Sequence, output_sequence_length: Optional[int] = None,
              lower: bool = True, strip: bool = True) -> np.ndarray:
  """int64 [B, T]: 0 padding, 1 OOV, vocabulary[i] -> 2 + i (entries compared as bytes, not standardized)."""
  index: Dict[bytes, int] = {as_bytes(v): 2 + i for i, v in enumerate(vocabulary)}
  toks = [tokens(s, lower, strip) for s in strings]
  T = output_sequence_length if output_sequence_length is not None else max([len(t) for t in toks], default=0)
  out = np.zeros((len(toks), T), np.int64)
  for b, ts in enumerate(toks):
    for j, t in enumerate(ts[:T]):
      out[b, j] = index.get(t, 1)
  return out


def adapt_vocabulary(strings: Sequence, max_tokens: Optional[int] = None, lower: bool = True,
                     strip: bool = True) -> List[bytes]:
  """Count descending, ties by token descending bytewise (tf-keras: np.lexsort((tokens, counts))[::-1]), cut to
  max_tokens - 2."""
  counts: Dict[bytes, int] = {}
  for s in strings:
    for t in tokens(s, lower, strip):
      counts[t] = counts.get(t, 0) + 1
  toks = list(counts)
  order = np.lexsort((np.array(toks, dtype=object), np.array([counts[t] for t in toks])))[::-1] if toks else []
  vocab = [toks[i] for i in order]
  return vocab if max_tokens is None else vocab[:max(max_tokens - 2, 0)]


# ---- Discretization --------------------------------------------------------------------------------------------------
def bucketize(x: np.ndarray, boundaries: Sequence[float]) -> np.ndarray:
  """#{i : f32(b_i) <= x} (std::upper_bound); integers rounded to float32 first, float64 compared as doubles, NaN last."""
  b = np.asarray(boundaries, np.float64).astype(np.float32)
  x = np.asarray(x)
  if x.dtype == np.float64:
    v, bb = x, b.astype(np.float64)
  else:
    v, bb = x.astype(np.float32), b
  out = np.searchsorted(bb, v.reshape(-1), side="right").astype(np.int64)
  out[np.isnan(v.reshape(-1))] = len(b)
  return out.reshape(x.shape)


# ---- Normalization ---------------------------------------------------------------------------------------------------
def _std(variance) -> np.ndarray:
  return np.maximum(np.sqrt(np.float32(variance)), EPSILON)


def normalize(x: np.ndarray, mean, variance, invert: bool = False) -> np.ndarray:
  x = np.asarray(x).astype(np.float32)
  m, sd = np.float32(mean), _std(variance)
  with np.errstate(all="ignore"):
    return (m + x * sd) if invert else ((x - m) / sd)


def _sum64(v: np.ndarray) -> np.float64:
  """The float64 sum in element order, one addition at a time (np.cumsum is sequential)."""
  return np.cumsum(v.astype(np.float64))[-1] if v.size else np.float64(0)


def batch_moments(x: np.ndarray, C: int):
  """float32 [C] mean and variance of one batch: x [rows, ...], channel = last index mod C, row-major element order."""
  x = np.asarray(x).astype(np.float32).reshape(x.shape[0], -1)
  means, variances = np.zeros(C, np.float32), np.zeros(C, np.float32)
  for c in range(C):
    v = x[:, c::C].reshape(-1)
    n = np.float64(v.size)
    m = np.float32(_sum64(v) / n)
    d = v - m
    means[c], variances[c] = m, np.float32(_sum64(d * d) / n)
  return means, variances, x.shape[0] * (x.shape[1] // C)


def merge(mean, var, total, mb, vb, nb):
  """Keras's Normalization.update_state merge, one float32 operation at a time."""
  total = total + nb
  w = np.float32(nb) / np.float32(total)
  ew = np.float32(1) - w
  nm = mean * ew + mb * w
  d0, d1 = mean - nm, mb - nm
  with np.errstate(all="ignore"):
    nv = (var + d0 * d0) * ew + (vb + d1 * d1) * w
  return nm.astype(np.float32), nv.astype(np.float32), total


def adapt_moments(batches: Sequence[np.ndarray], C: int):
  """(mean, variance) float32 [C] after merging the batches in order from Keras's initial state (0, 1, count 0)."""
  mean, var, total = np.zeros(C, np.float32), np.ones(C, np.float32), 0
  for x in batches:
    x = np.asarray(x)
    x = x.reshape(1) if x.ndim == 0 else x
    if x.shape[0] == 0:
      continue
    mb, vb, nb = batch_moments(x, C)
    mean, var, total = merge(mean, var, total, mb, vb, nb)
  return mean, var


def array_batches(x: np.ndarray, batch_size: int = 32) -> List[np.ndarray]:
  return [x[i:i + batch_size] for i in range(0, x.shape[0], batch_size)]


# ---- GlobalAveragePooling1D ------------------------------------------------------------------------------------------
def pool(x: np.ndarray, mask: Optional[np.ndarray] = None) -> np.ndarray:
  """[B, d]: sum_t f32(x * m) sequentially from +0.0f over sum_t m, or sum_t x / T."""
  x = np.asarray(x, np.float32)
  B, T, d = x.shape
  s = np.zeros((B, d), np.float32)
  with np.errstate(all="ignore"):
    if mask is None:
      for t in range(T):
        s = s + x[:, t]
      return s / np.float32(T)
    m = (np.asarray(mask) != 0).astype(np.float32)
    for t in range(T):
      s = s + x[:, t] * m[:, t, None]
    return s / m.sum(axis=1, dtype=np.float32)[:, None]


def pool_grad(g: np.ndarray, mask: Optional[np.ndarray], T: int) -> np.ndarray:
  """[B, T, d]: f32(g / count) * m, or g / T."""
  g = np.asarray(g, np.float32)
  with np.errstate(all="ignore"):
    if mask is None:
      return np.repeat((g / np.float32(T))[:, None, :], T, axis=1)
    m = (np.asarray(mask) != 0).astype(np.float32)
    q = g / m.sum(axis=1, dtype=np.float32)[:, None]
    return q[:, None, :] * m[:, :, None]


# ---- constants read back from the kernel source ----------------------------------------------------------------------
def kernel_byte_sets() -> Dict[str, bytes]:
  """The punctuation and whitespace bytes csrc/text.cu compiles in (TX_PUNCT, TX_SPACE)."""
  src = open(os.path.join(ROOT, "recommenders_b200", "csrc", "text.cu")).read()
  out = {}
  for name in ("TX_PUNCT", "TX_SPACE"):
    body = re.search(rf"constexpr uint8_t {name}\[(\d+)\] = \{{(.*?)\}};", src, re.S)
    vals = bytes(int(v, 16) for v in re.findall(r"0x[0-9a-fA-F]{2}", body.group(2)))
    assert len(vals) == int(body.group(1)), name
    out[name] = vals
  return out
