"""Host-side packing of string inputs (NumPy str / bytes / object arrays, or lists) into one byte buffer with int64
offsets, the layout the C ABI takes for TFRS_BYTES values.  Shared by UnifiedEmbedding and the lookup layers."""
from __future__ import annotations

from typing import Tuple

import numpy as np
import torch


def pack_strings(values) -> Tuple[np.ndarray, np.ndarray, Tuple[int, ...]]:
  """(UTF-8 bytes of every string back to back, int64 offsets [n+1], shape), vectorised over the array."""
  a = np.asarray(values)
  if a.dtype.kind == "O":
    first = next(iter(a.flat), "")
    a = a.astype("S" if isinstance(first, (bytes, np.bytes_)) else "U")
  if a.dtype.kind == "U":
    flat = np.ascontiguousarray(a.reshape(-1))
    width = flat.dtype.itemsize // 4
    cp = flat.view(np.uint32).reshape(flat.size, width) if flat.size and width else None
    if cp is not None and int(cp.max()) < 0x80:
      # all ASCII: UTF-8 is one byte per code point, so the bytes come straight from the UCS-4 array
      lens = np.char.str_len(flat).astype(np.int64)
      offsets = np.zeros(flat.size + 1, np.int64)
      np.cumsum(lens, out=offsets[1:])
      return cp[np.arange(width) < lens[:, None]].astype(np.uint8), offsets, a.shape
    a = np.char.encode(a, "utf-8")
  flat = np.ascontiguousarray(a.reshape(-1))
  lens = np.char.str_len(flat).astype(np.int64) if flat.size else np.zeros(0, np.int64)
  offsets = np.zeros(flat.size + 1, np.int64)
  np.cumsum(lens, out=offsets[1:])
  w = flat.dtype.itemsize
  if flat.size == 0 or w == 0:
    return np.zeros(0, np.uint8), offsets, a.shape
  data = flat.view(np.uint8).reshape(flat.size, w)[np.arange(w) < lens[:, None]]
  return data, offsets, a.shape


def is_strings(x) -> bool:
  if isinstance(x, np.ndarray):
    return x.dtype.kind in "USO"
  return isinstance(x, list) and len(x) > 0 and isinstance(x[0], (str, bytes))


def upload_packed(data: np.ndarray, offsets: np.ndarray, device, extra: np.ndarray = None):
  """(uint8 bytes, int64 offsets) on `device` after ONE host-to-device copy: the offsets first (8-byte aligned), then the
  bytes, then `extra` bytes (returned as a third tensor when given)."""
  parts = [offsets.view(np.uint8), data] + ([extra] if extra is not None else [])
  dev = torch.from_numpy(np.concatenate(parts)).to(device)
  n64, nb = offsets.size, data.size
  offs = dev[:8 * n64].view(torch.int64)
  byts = dev[8 * n64:8 * n64 + nb] if nb else dev[:0]
  if extra is None:
    return byts, offs
  return byts, offs, dev[8 * n64 + nb:]
