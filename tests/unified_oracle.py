"""CPU oracle of UnifiedEmbedding (layers/feature_multiplexing/unified_embedding.py) and of tf-keras `Hashing` with a salt.

Test infrastructure, like clippy_oracle.py: the product never imports it.  The hashing, the lookups and the pooling are
plain C (unified_oracle.c, compiled by `build()` -- which __graft_entry__.build() calls -- into libunified_oracle.so
next to it) so the GPU tests can compare millions of hashes; the layer bookkeeping (table round-robin, salts, the
sorted() order of the chunk names) is restated below from unified_embedding.py:98-126,199-215, independently of recommenders_b200.
"""
from __future__ import annotations

import ctypes
import os
import subprocess
from typing import Dict, List, Sequence, Tuple

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "unified_oracle.c")
_LIB = None
COMBINERS = {"sum": 0, "mean": 1, "sqrtn": 2}
_u64, _i64, _p = ctypes.c_uint64, ctypes.c_int64, ctypes.c_void_p


def build(force: bool = False) -> str:
  """Compiles unified_oracle.c -> libunified_oracle.so beside it (no FMA contraction, no fast-math); returns the path."""
  so = os.path.join(_HERE, "libunified_oracle.so")
  if force or not os.path.exists(so) or os.path.getmtime(so) < os.path.getmtime(_SRC):
    subprocess.check_call([os.environ.get("CC", "cc"), "-O2", "-ffp-contract=off", "-fno-fast-math", "-shared", "-fPIC",
                           _SRC, "-o", so, "-lm"])
  return so


def _lib() -> ctypes.CDLL:
  global _LIB
  if _LIB is None:
    lib = ctypes.CDLL(build())
    lib.uo_siphash.restype = _u64
    lib.uo_siphash.argtypes = [_u64, _u64, _p, _i64]
    lib.uo_as_string.restype = ctypes.c_int
    lib.uo_as_string.argtypes = [_i64, ctypes.c_char_p]
    lib.uo_hash_i64.argtypes = [_p, _i64, _u64, _u64, _u64, _p]
    lib.uo_hash_bytes.argtypes = [_p, _p, _i64, _u64, _u64, _u64, _p]
    lib.uo_gather.argtypes = [_p, ctypes.c_int, _p, _i64, _p, _i64, _i64]
    lib.uo_pool.argtypes = [_p, ctypes.c_int, _p, _p, _i64, ctypes.c_int, _p, _i64, _i64]
    lib.uo_pool_bwd.argtypes = [_p, _i64, _i64, ctypes.c_int, _p, _i64, ctypes.c_int, _p]
    _LIB = lib
  return _LIB


def _ptr(a: np.ndarray):
  return a.ctypes.data_as(ctypes.c_void_p)


def salt_key(salt) -> Tuple[int, int]:
  """tf-keras Hashing: an int salt s is the key [s, s]."""
  if isinstance(salt, (int, np.integer)):
    salt = (salt, salt)
  return int(salt[0]) & (2**64 - 1), int(salt[1]) & (2**64 - 1)


def siphash(k0: int, k1: int, msg: bytes) -> int:
  buf = np.frombuffer(msg, np.uint8).copy() if msg else np.zeros(1, np.uint8)
  return int(_lib().uo_siphash(k0, k1, _ptr(buf), len(msg)))


def as_string(x: int) -> bytes:
  buf = ctypes.create_string_buffer(24)
  n = _lib().uo_as_string(int(x), buf)
  return buf.raw[:n]


def is_string_array(values) -> bool:
  if isinstance(values, np.ndarray):
    return values.dtype.kind in "USO"
  return isinstance(values, (list, tuple)) and (not values or isinstance(values[0], (str, bytes)))


def pack(values) -> Tuple[np.ndarray, np.ndarray]:
  """UTF-8 bytes of every string (bytes as given) and int64 offsets [n+1]; one Python loop, this is the oracle."""
  items = [v.encode("utf-8") if isinstance(v, str) else bytes(v) for v in np.asarray(values, dtype=object).reshape(-1)]
  off = np.zeros(len(items) + 1, np.int64)
  off[1:] = np.cumsum([len(b) for b in items])
  data = np.frombuffer(b"".join(items), np.uint8).copy() if off[-1] else np.zeros(1, np.uint8)
  return data, off


def hash_bins(values, num_bins: int, salt) -> np.ndarray:
  """to_hash_bucket_strong(as_string(values) or values, num_bins, key=salt_key(salt)), int64, values' shape."""
  k0, k1 = salt_key(salt)
  if is_string_array(values):
    shape = np.asarray(values, dtype=object).shape
    data, off = pack(values)
    out = np.empty(len(off) - 1, np.int64)
    _lib().uo_hash_bytes(_ptr(data), _ptr(off), len(out), k0, k1, int(num_bins), _ptr(out))
    return out.reshape(shape)
  v = np.ascontiguousarray(values, dtype=np.int64)
  out = np.empty(v.shape, np.int64)
  _lib().uo_hash_i64(_ptr(v), v.size, k0, k1, int(num_bins), _ptr(out))
  return out


def plan(spec: Sequence[Tuple[str, int]], num_tables: int, name: str):
  """[(feature, [(chunk_id, table, salt, column slot)])]: UnifiedEmbeddingConfig.add_feature's round-robin table cursor
  (carried across features) and salt [feature_index, chunk_id]; the column slot is the chunk name's rank in sorted()."""
  cur, out = 0, []
  for fi, (feat, nc) in enumerate(spec):
    names = [f"{name}_{feat}_lookup_{c}" for c in range(nc)]
    order = sorted(names)
    chunks = []
    for c in range(nc):
      chunks.append((c, cur, (fi, c), order.index(names[c])))
      cur = (cur + 1) % num_tables
    out.append((feat, chunks))
  return out


def forward(features: Dict, spec, tables: Sequence[np.ndarray], name: str, combiner: str = "mean"):
  """UnifiedEmbedding.call: (list of outputs, {table: bucket ids in config order}).  A (values, row_splits) feature is
  pooled with `combiner`; any other is looked up value by value (shape [..., width])."""
  dim = tables[0].shape[1]
  outs, ids = [], {t: [] for t in range(len(tables))}
  for feat, chunks in plan(spec, len(tables), name):
    x = features[feat]
    ragged = isinstance(x, tuple)
    values = x[0] if ragged else x
    flat = np.asarray(values, dtype=object if is_string_array(values) else np.int64).reshape(-1)
    width = len(chunks) * dim
    rows = len(x[1]) - 1 if ragged else flat.size
    out = np.zeros((rows, width), np.float32)
    for c, t, salt, pos in chunks:
      tab = np.ascontiguousarray(tables[t], np.float32)
      b = np.ascontiguousarray(hash_bins(flat, tab.shape[0], salt).reshape(-1))
      ids[t].append(b)
      if ragged:
        sp = np.ascontiguousarray(x[1], np.int64)
        _lib().uo_pool(_ptr(tab), dim, _ptr(b), _ptr(sp), rows, COMBINERS[combiner], _ptr(out), width, pos * dim)
      else:
        _lib().uo_gather(_ptr(tab), dim, _ptr(b), rows, _ptr(out), width, pos * dim)
    outs.append(out if ragged else out.reshape(*np.shape(values), width))
  return outs, {t: np.concatenate(v) for t, v in ids.items() if v}


def backward(features: Dict, spec, num_tables: int, dim: int, name: str, grads: Sequence[np.ndarray],
             combiner: str = "mean") -> Dict[int, np.ndarray]:
  """The gradient rows of each table, in the order of forward's ids: a lookup's row gets its output gradient, a pooled
  value its bag's gradient divided as in the forward."""
  rows = {t: [] for t in range(num_tables)}
  for (feat, chunks), g in zip(plan(spec, num_tables, name), grads):
    x = features[feat]
    width = len(chunks) * dim
    g = np.ascontiguousarray(g, np.float32).reshape(-1, width)
    for c, t, salt, pos in chunks:
      if isinstance(x, tuple):
        sp = np.ascontiguousarray(x[1], np.int64)
        r = np.zeros((int(sp[-1]), dim), np.float32)
        _lib().uo_pool_bwd(_ptr(g), width, pos * dim, dim, _ptr(sp), len(sp) - 1, COMBINERS[combiner], _ptr(r))
      else:
        r = g[:, pos * dim:(pos + 1) * dim].copy()
      rows[t].append(r)
  return {t: np.concatenate(v) for t, v in rows.items() if v}
