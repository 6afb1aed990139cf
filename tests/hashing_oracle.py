"""CPU oracle of tf-keras `Hashing` (K18, recommenders_b200/csrc/hashing.cu), salted or not, with or without a mask.

Test infrastructure: the product never imports it.  The hashing is plain C (hashing_oracle.c, compiled by `build()` --
which __graft_entry__.build() calls -- together with unified_oracle.c, whose SipHash and tf.as_string it uses, into
libhashing_oracle.so next to it).  String packing and salt keys are unified_oracle's.
"""
from __future__ import annotations

import ctypes
import os
import subprocess

import numpy as np

import unified_oracle as uo

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRCS = [os.path.join(_HERE, "hashing_oracle.c"), os.path.join(_HERE, "unified_oracle.c")]
_LIB = None
_u64, _i64, _p, _int = ctypes.c_uint64, ctypes.c_int64, ctypes.c_void_p, ctypes.c_int


def build(force: bool = False) -> str:
  """Compiles hashing_oracle.c and unified_oracle.c -> libhashing_oracle.so beside them; returns the path."""
  so = os.path.join(_HERE, "libhashing_oracle.so")
  if force or not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(s) for s in _SRCS):
    subprocess.check_call([os.environ.get("CC", "cc"), "-O2", "-shared", "-fPIC", *_SRCS, "-o", so, "-lm"])
  return so


def _lib() -> ctypes.CDLL:
  global _LIB
  if _LIB is None:
    lib = ctypes.CDLL(build())
    lib.ho_fingerprint64.restype = _u64
    lib.ho_fingerprint64.argtypes = [_p, _i64]
    lib.ho_hash_i64.argtypes = [_p, _i64, _int, _u64, _u64, _u64, _int, _i64, _p]
    lib.ho_hash_bytes.argtypes = [_p, _p, _i64, _int, _u64, _u64, _u64, _int, _p, _i64, _p]
    _LIB = lib
  return _LIB


def _ptr(a: np.ndarray):
  return a.ctypes.data_as(ctypes.c_void_p)


def fingerprint64(msg: bytes) -> int:
  """FarmHash Fingerprint64 (farmhashna::Hash64) of `msg`, as TF's Fingerprint64."""
  buf = np.frombuffer(msg, np.uint8).copy() if msg else np.zeros(1, np.uint8)
  return int(_lib().ho_fingerprint64(_ptr(buf), len(msg)))


def _as_bytes(v) -> bytes:
  return v.encode("utf-8") if isinstance(v, str) else bytes(v)


def hashing(values, num_bins: int, salt=None, mask=None) -> np.ndarray:
  """tf-keras Hashing(num_bins, mask_value=mask, salt=salt)(values): int64 in values' shape.  Strings (str as UTF-8, or
  bytes) hash as their bytes, integers as their tf.as_string text."""
  salted = salt is not None
  k0, k1 = uo.salt_key(salt) if salted else (0, 0)
  if uo.is_string_array(values):
    shape = np.asarray(values, dtype=object).shape
    data, off = uo.pack(values)
    out = np.empty(len(off) - 1, np.int64)
    m = np.frombuffer(_as_bytes(mask), np.uint8).copy() if mask is not None else np.zeros(0, np.uint8)
    mbuf = m if m.size else np.zeros(1, np.uint8)
    _lib().ho_hash_bytes(_ptr(data), _ptr(off), len(out), int(salted), k0, k1, int(num_bins), int(mask is not None),
                         _ptr(mbuf), m.size, _ptr(out))
    return out.reshape(shape)
  v = np.ascontiguousarray(values, dtype=np.int64)
  out = np.empty(v.shape, np.int64)
  _lib().ho_hash_i64(_ptr(v), v.size, int(salted), k0, k1, int(num_bins), int(mask is not None),
                     0 if mask is None else int(mask), _ptr(out))
  return out
