"""Functional wrappers over the C ABI (one Python function per entry point of include/tfrs_b200.h).

Everything here takes/returns CUDA torch tensors; torch only provides memory, streams and the
autograd tape.  No CPU fallback.
"""
from __future__ import annotations

import ctypes
import math
from typing import NamedTuple, Optional, Sequence, Tuple

import numpy as np
import torch

from . import _ffi
from ._ffi import c_f, c_i, c_l, c_p, c_sz, check, f32c, lib, ptr, require_cuda, stream, workspace

# Corpora at least this large go through the tensor-core screening path when an index image exists.
TC_MIN_N = 16384
TC_MAX_K = 256
TC_MAX_Q_PER_CALL = 8192


# ------------------------------------------------------------------------------------------------
# K1 gather
# ------------------------------------------------------------------------------------------------
def gather(tables: Sequence[torch.Tensor], ids: Sequence[torch.Tensor], out: Optional[torch.Tensor] = None,
           col_offsets: Optional[Sequence[int]] = None) -> torch.Tensor:
  """out[i, off_t:off_t+dim_t] = tables[t][ids[t][i]]  -- concatenated multi-table embedding lookup."""
  nt = len(tables)
  if nt == 0 or len(ids) != nt:
    raise ValueError("gather: need as many id tensors as tables")
  n = ids[0].numel()
  dims = [int(t.shape[1]) for t in tables]
  if col_offsets is None:
    col_offsets, o = [], 0
    for d in dims:
      col_offsets.append(o); o += d
    width = o
  else:
    width = max(o + d for o, d in zip(col_offsets, dims))
  dev = tables[0].device
  tabs = [f32c(t, "table") for t in tables]
  code = _ffi.ids_dtype_code(ids[0])
  idl = []
  for x in ids:
    require_cuda(x, "ids")
    if _ffi.ids_dtype_code(x) != code or x.numel() != n:
      raise ValueError("gather: all id tensors must share dtype and length")
    idl.append(x.contiguous().view(-1))
  if out is None:
    out = torch.empty((n, width), dtype=torch.float32, device=dev)
  else:
    require_cuda(out, "out")
    if out.dtype != torch.float32 or out.stride(-1) != 1 or out.shape[0] != n:
      raise ValueError("gather: out must be float32 [n, >=width] with unit inner stride")
  out_ld = out.stride(0) if out.dim() == 2 else width
  tp = (ctypes.c_void_p * nt)(*[t.data_ptr() for t in tabs])
  ip = (ctypes.c_void_p * nt)(*[x.data_ptr() for x in idl])
  rows = (ctypes.c_int64 * nt)(*[int(t.shape[0]) for t in tabs])
  dm = (ctypes.c_int32 * nt)(*dims)
  co = (ctypes.c_int32 * nt)(*[int(c) for c in col_offsets])
  check(lib().tfrs_gather_f32(tp, rows, dm, nt, ip, code, n, ptr(out), out_ld, co, stream()), "gather")
  return out


# ------------------------------------------------------------------------------------------------
# K8 UnifiedEmbedding: salted SipHash bucketing fused with the shared-table gather
# ------------------------------------------------------------------------------------------------
COMBINERS = {"sum": 0, "mean": 1, "sqrtn": 2}


class _UeFeature(ctypes.Structure):
  _fields_ = [("values", ctypes.c_void_p), ("offsets", ctypes.c_void_p), ("n", ctypes.c_int64),
              ("row_splits", ctypes.c_void_p), ("n_bags", ctypes.c_int64), ("kind", ctypes.c_int32),
              ("combiner", ctypes.c_int32), ("n_chunks", ctypes.c_int32), ("reserved", ctypes.c_int32)]


class _UeSlot(ctypes.Structure):
  _fields_ = [("table", ctypes.c_void_p), ("rows", ctypes.c_int64), ("salt", ctypes.c_uint64 * 2),
              ("out", ctypes.c_void_p), ("ld", ctypes.c_int64), ("col_off", ctypes.c_int32), ("dim", ctypes.c_int32),
              ("ids", ctypes.c_void_p), ("grad", ctypes.c_void_p), ("grad_rows", ctypes.c_void_p)]


def salt_key(salt) -> Tuple[int, int]:
  """The SipHash key of a tf-keras `Hashing` salt: an int s means (s, s), a pair is (k0, k1); both as uint64."""
  if isinstance(salt, int):
    salt = (salt, salt)
  k0, k1 = (int(s) for s in salt)
  return k0 & (2**64 - 1), k1 & (2**64 - 1)


class LookupInput(NamedTuple):
  """One input stream: CUDA int32 / int64 `values`, or the uint8 bytes of strings with their int64 `offsets` [n+1].
  `row_splits` (int64 [bags+1]) pools the values into bags with `combiner`."""
  values: torch.Tensor
  offsets: Optional[torch.Tensor] = None
  row_splits: Optional[torch.Tensor] = None
  combiner: str = "mean"

  @property
  def n(self) -> int:
    return self.values.numel() if self.offsets is None else self.offsets.numel() - 1


class LookupSlot(NamedTuple):
  """One (feature, chunk) lookup: `table` [num_bins, dim] hashed with `salt`, written to columns [col_off, col_off+dim)
  of the 2-D `out`; the bucket ids go to `ids` (int64 [n]) when it is given (required for pooled inputs)."""
  input: int
  table: torch.Tensor
  salt: Tuple[int, int]
  out: torch.Tensor
  col_off: int
  ids: Optional[torch.Tensor] = None


def _value_kind(values: torch.Tensor, offsets: Optional[torch.Tensor]) -> int:
  require_cuda(values, "values")
  if offsets is not None:
    require_cuda(offsets, "offsets")
    if values.dtype != torch.uint8 or offsets.dtype != torch.int64:
      raise TypeError("string values must be uint8 bytes with int64 offsets")
    return _ffi.BYTES
  return _ffi.ids_dtype_code(values)


def hash_bins(values, num_bins: int, salt) -> torch.Tensor:
  """tf-keras `Hashing(num_bins, salt=salt)` on the device: SipHash-2-4 keyed by the salt, mod num_bins, int64.  `values`
  is a CUDA int32 / int64 tensor (hashed as its decimal text) or a (uint8 bytes, int64 offsets [n+1]) pair of strings."""
  values, offsets = values if isinstance(values, tuple) else (values, None)
  kind = _value_kind(values, offsets)
  values = values.contiguous()
  offsets = offsets.contiguous() if offsets is not None else None
  n = values.numel() if offsets is None else offsets.numel() - 1
  out = torch.empty(values.shape if offsets is None else (n,), dtype=torch.int64, device=values.device)
  key = (ctypes.c_uint64 * 2)(*salt_key(salt))
  check(lib().tfrs_hash_bins(ptr(values), ptr(offsets), kind, n, key, int(num_bins), ptr(out), stream()), "hash_bins")
  return out


# ------------------------------------------------------------------------------------------------
# K18 feature hashing: layers.Hashing
# ------------------------------------------------------------------------------------------------
def hashing(values, num_bins: int, salt=None, mask=None) -> torch.Tensor:
  """tf-keras `Hashing(num_bins, mask_value=mask, salt=salt)` on the device, int64 in the values' shape (1-D for strings).
  `values` is a CUDA int32 / int64 tensor (hashed as its decimal text) or a (uint8 bytes, int64 offsets [n+1]) pair of
  CUDA tensors.  Without a salt the hash is FarmHash Fingerprint64 (`to_hash_bucket_fast`), with one SipHash-2-4 keyed
  by `salt_key(salt)`.  `mask` is an int for integer values or a CUDA uint8 tensor of the mask string's bytes; with
  num_bins > 1 it takes bin 0 and every other value 1 + h mod (num_bins - 1).  One launch."""
  values, offsets = values if isinstance(values, tuple) else (values, None)
  kind = _value_kind(values, offsets)
  if isinstance(num_bins, bool) or not isinstance(num_bins, (int, np.integer)) or not 1 <= num_bins < 2**63:
    raise ValueError(f"hashing: num_bins must be an int in [1, 2^63), got {num_bins!r}")
  values = values.contiguous()
  offsets = offsets.contiguous() if offsets is not None else None
  n = values.numel() if offsets is None else offsets.numel() - 1
  out = torch.empty(values.shape if offsets is None else (n,), dtype=torch.int64, device=values.device)
  key = None if salt is None else (ctypes.c_uint64 * 2)(*salt_key(salt))
  mask_int, mask_bytes = 0, None
  if mask is not None:
    if offsets is None:
      if isinstance(mask, (bool, torch.Tensor)) or not isinstance(mask, (int, np.integer)):
        raise TypeError(f"hashing: the mask of integer values must be an int, got {mask!r}")
      if not -2**63 <= int(mask) < 2**63:
        raise ValueError(f"hashing: the mask {mask} does not fit in int64")
      mask_int = int(mask)
    else:
      require_cuda(mask, "mask")
      if mask.dtype != torch.uint8:
        raise TypeError("hashing: the mask of string values must be uint8 bytes")
      mask_bytes = mask.contiguous()
  check(lib().tfrs_hashing(ptr(values), ptr(offsets), kind, n, key, int(num_bins), int(mask is not None), mask_int,
                           ptr(mask_bytes), 0 if mask_bytes is None else mask_bytes.numel(), ptr(out), stream()),
        "hashing")
  return out


def _out_rows(x: LookupInput) -> int:
  return x.n if x.row_splits is None else x.row_splits.numel() - 1


def _check_2d(t: torch.Tensor, rows: int, what: str, op: str) -> None:
  require_cuda(t, what)
  if t.dtype != torch.float32 or t.dim() != 2 or t.shape[0] != rows or (t.stride(1) != 1 and t.numel() > 0):
    raise ValueError(f"{op}: {what} must be 2-D float32 [{rows}, >= width] with unit inner stride")


def _view_ld(m: torch.Tensor, col_off: int, dim: int, what: str, op: str) -> int:
  """The row stride (`ld`) the kernels use for columns [col_off, col_off + dim) of the 2-D view `m` (checked by
  _check_2d): its stride(0), or its width when it has at most one row.  Columns past the view's width, and rows that
  overlap (0 < stride(0) < width, or an expanded view with stride(0) == 0), raise: the kernel would read or write
  outside the view, and past its storage on the last row."""
  width = m.shape[1]
  if col_off < 0 or col_off + dim > width:
    raise ValueError(f"{op}: {what}: columns [{col_off}, {col_off + dim}) run outside its {width} columns")
  if m.shape[0] <= 1:
    return width
  if m.stride(0) < width:
    raise ValueError(f"{op}: {what}: rows overlap (row stride {m.stride(0)} < width {width}); pass a contiguous tensor")
  return m.stride(0)


def _check_splits(s: torch.Tensor, op: str) -> None:
  require_cuda(s, "row_splits")
  if s.dtype != torch.int64 or s.dim() != 1 or s.numel() < 1:
    raise TypeError("row_splits must be a non-empty 1-D int64 tensor")
  if not s.is_contiguous():
    raise ValueError(f"{op}: row_splits must be contiguous")


def _check_table(t: torch.Tensor, op: str) -> None:
  require_cuda(t, "table")
  if t.dtype != torch.float32 or not t.is_contiguous() or t.dim() != 2:
    raise ValueError(f"{op}: tables must be contiguous 2-D float32")


def _check_ids(ids: torch.Tensor, n: int, op: str) -> None:
  require_cuda(ids, "ids")
  if ids.dtype != torch.int64 or not ids.is_contiguous() or ids.numel() != n:
    raise ValueError(f"{op}: ids must be contiguous int64 with one entry per value")


def _check_grad_rows(r: torch.Tensor, n: int, dim: int, op: str) -> None:
  require_cuda(r, "grad_rows")
  if r.dtype != torch.float32 or not r.is_contiguous() or r.shape != (n, dim):
    raise ValueError(f"{op}: grad_rows must be contiguous float32 [n, dim]")


def _ue_structs(inputs: Sequence[LookupInput], slots: Sequence[LookupSlot], outs: Sequence[torch.Tensor]):
  """The C descriptors of one call; slots must come grouped by input, inputs in order.  `outs[c]` is the 2-D tensor
  slot c's columns live in: its output in the forward, the gradient of that output in the backward."""
  order = [s.input for s in slots]
  if order != sorted(order) or set(order) != set(range(len(inputs))):
    raise ValueError("unified_lookup: every input needs slots, grouped by input in input order")
  counts = [order.count(k) for k in range(len(inputs))]
  feats = (_UeFeature * len(inputs))()
  for k, x in enumerate(inputs):
    f = feats[k]
    f.kind = _value_kind(x.values, x.offsets)
    f.values, f.offsets = x.values.data_ptr(), (x.offsets.data_ptr() if x.offsets is not None else None)
    f.n, f.n_chunks = x.n, counts[k]
    if x.row_splits is not None:
      _check_splits(x.row_splits, "unified_lookup")
      f.row_splits, f.n_bags, f.combiner = x.row_splits.data_ptr(), x.row_splits.numel() - 1, COMBINERS[x.combiner]
  cs = (_UeSlot * len(slots))()
  for c, (s, o) in enumerate(zip(slots, outs)):
    _check_table(s.table, "unified_lookup")
    _check_2d(o, _out_rows(inputs[s.input]), "each output / gradient", "unified_lookup")
    d = cs[c]
    d.table, d.rows, d.dim = s.table.data_ptr(), s.table.shape[0], s.table.shape[1]
    d.salt[0], d.salt[1] = s.salt
    d.ld, d.col_off = _view_ld(o, s.col_off, d.dim, "each output / gradient", "unified_lookup"), s.col_off
    if s.ids is not None:
      _check_ids(s.ids, inputs[s.input].n, "unified_lookup")
      d.ids = s.ids.data_ptr()
  return feats, cs


def unified_lookup(inputs: Sequence[LookupInput], slots: Sequence[LookupSlot]) -> None:
  """Every (feature, chunk) lookup of one UnifiedEmbedding call: out[:, col_off:col_off+dim] = table[bin(value)], or the
  pooled bag of rows for inputs with row_splits.  One launch (two with pooled inputs)."""
  feats, cs = _ue_structs(inputs, slots, [s.out for s in slots])
  for c, s in enumerate(slots):
    cs[c].out = s.out.data_ptr()
  check(lib().tfrs_unified_lookup_fwd_f32(feats, len(inputs), cs, len(slots), stream()), "unified_lookup")


def unified_lookup_bwd(inputs: Sequence[LookupInput], slots: Sequence[LookupSlot], grads: Sequence[torch.Tensor],
                       grad_rows: Sequence[torch.Tensor]) -> None:
  """grad_rows[c] ([n, dim]) = the gradient of slot c's table rows, value by value: grads[c] (the gradient of the 2-D
  output slot c wrote into; `slots[c].out` itself is not read) at the slot's columns, divided by the combiner for pooled
  inputs.  One launch."""
  if len(grads) != len(slots) or len(grad_rows) != len(slots):
    raise ValueError("unified_lookup_bwd: one gradient and one grad_rows tensor per slot")
  feats, cs = _ue_structs(inputs, slots, grads)
  for c, (g, r) in enumerate(zip(grads, grad_rows)):
    _check_grad_rows(r, inputs[slots[c].input].n, cs[c].dim, "unified_lookup_bwd")
    cs[c].grad, cs[c].grad_rows = g.data_ptr(), r.data_ptr()
  check(lib().tfrs_unified_lookup_bwd_f32(feats, len(inputs), cs, len(slots), stream()), "unified_lookup_bwd")


# ------------------------------------------------------------------------------------------------
# K11 weighted multi-hot bag pooling (TPUEmbedding)
# ------------------------------------------------------------------------------------------------
class _BagFeature(ctypes.Structure):
  _fields_ = [("table", ctypes.c_void_p), ("rows", ctypes.c_int64), ("dim", ctypes.c_int32), ("kind", ctypes.c_int32),
              ("values", ctypes.c_void_p), ("n", ctypes.c_int64), ("row_splits", ctypes.c_void_p),
              ("n_bags", ctypes.c_int64), ("weights", ctypes.c_void_p), ("combiner", ctypes.c_int32),
              ("max_seq_len", ctypes.c_int32), ("out", ctypes.c_void_p), ("ld", ctypes.c_int64),
              ("col_off", ctypes.c_int32), ("reserved", ctypes.c_int32), ("ids", ctypes.c_void_p),
              ("denom", ctypes.c_void_p), ("grad", ctypes.c_void_p), ("grad_rows", ctypes.c_void_p)]


class BagFeature(NamedTuple):
  """One feature of an embedding_bag call.  `values`: CUDA int32 / int64 ids (flattened).  With `row_splits` (int64
  [bags+1]) the values form bags: pooled with `combiner`, or, when `max_sequence_length` L > 0, laid out as L positions
  per bag.  Without, every value is looked up on its own (dense).  `weights` (fp32, one per value) only with bags.
  `out` is 2-D with one row per output row (bags, bags * L, or values); this feature's columns are
  [col_off, col_off + dim).  `ids` (int64 [n]) receives the ids for the backward pair; `denom` (fp32 [bags]) receives
  the mean / sqrtn denominators, which the backward needs."""
  table: torch.Tensor
  values: torch.Tensor
  out: torch.Tensor
  row_splits: Optional[torch.Tensor] = None
  weights: Optional[torch.Tensor] = None
  combiner: str = "mean"
  max_sequence_length: int = 0
  col_off: int = 0
  ids: Optional[torch.Tensor] = None
  denom: Optional[torch.Tensor] = None


def bag_out_rows(f: BagFeature) -> int:
  if f.row_splits is None:
    return f.values.numel()
  bags = f.row_splits.numel() - 1
  return bags * f.max_sequence_length if f.max_sequence_length > 0 else bags


def _bag_structs(features: Sequence[BagFeature], mats: Sequence[torch.Tensor], op: str):
  """The C descriptors; `mats[k]` is the 2-D tensor feature k's columns live in (its output, or that output's gradient).
  `op` names the caller in error messages."""
  cs = (_BagFeature * len(features))()
  for k, (f, m) in enumerate(zip(features, mats)):
    d = cs[k]
    _check_table(f.table, "embedding_bag")
    d.table, d.rows, d.dim = f.table.data_ptr(), f.table.shape[0], f.table.shape[1]
    d.kind = _ffi.ids_dtype_code(require_cuda(f.values, "values"))
    if not f.values.is_contiguous():
      raise ValueError("embedding_bag: values must be contiguous")
    d.values, d.n = f.values.data_ptr(), f.values.numel()
    if f.row_splits is not None:
      _check_splits(f.row_splits, op)
      d.row_splits, d.n_bags = f.row_splits.data_ptr(), f.row_splits.numel() - 1
      d.combiner, d.max_seq_len = COMBINERS[f.combiner], int(f.max_sequence_length)
    if f.weights is not None:
      require_cuda(f.weights, "weights")
      if f.weights.dtype != torch.float32 or not f.weights.is_contiguous() or f.weights.numel() != f.values.numel():
        raise ValueError("embedding_bag: weights must be contiguous float32 with one entry per value")
      d.weights = f.weights.data_ptr()
    _check_2d(m, bag_out_rows(f), "each output / gradient", op)
    d.ld, d.col_off = _view_ld(m, f.col_off, d.dim, "each output / gradient", op), f.col_off
    if f.ids is not None:
      _check_ids(f.ids, f.values.numel(), "embedding_bag")
      d.ids = f.ids.data_ptr()
    if f.denom is not None:
      require_cuda(f.denom, "denom")
      if f.denom.dtype != torch.float32 or not f.denom.is_contiguous() or f.denom.numel() != d.n_bags:
        raise ValueError("embedding_bag: denom must be contiguous float32 with one entry per bag")
      d.denom = f.denom.data_ptr()
  return cs


def embedding_bag(features: Sequence[BagFeature]) -> None:
  """Every lookup of one call (tfrs_embedding_bag_fwd_f32): pooled bags, sequence positions and dense values written
  into each feature's `out`.  One launch for up to 128 features."""
  cs = _bag_structs(features, [f.out for f in features], "embedding_bag")
  for k, f in enumerate(features):
    cs[k].out = f.out.data_ptr()
  check(lib().tfrs_embedding_bag_fwd_f32(cs, len(features), stream()), "embedding_bag")


def embedding_bag_bwd(features: Sequence[BagFeature], grads: Sequence[torch.Tensor],
                      grad_rows: Sequence[torch.Tensor]) -> None:
  """grad_rows[k] ([n, dim]) = the gradient of feature k's table rows, value by value, from grads[k] (the gradient of
  its 2-D output; `out` itself is not read) and the forward's `denom`.  One launch for up to 128 features."""
  if len(grads) != len(features) or len(grad_rows) != len(features):
    raise ValueError("embedding_bag_bwd: one gradient and one grad_rows tensor per feature")
  cs = _bag_structs(features, grads, "embedding_bag_bwd")
  for k, (f, g, r) in enumerate(zip(features, grads, grad_rows)):
    _check_grad_rows(r, f.values.numel(), cs[k].dim, "embedding_bag_bwd")
    cs[k].grad, cs[k].grad_rows = g.data_ptr(), r.data_ptr()
  check(lib().tfrs_embedding_bag_bwd_f32(cs, len(features), stream()), "embedding_bag_bwd")


# ------------------------------------------------------------------------------------------------
# SGD (tf-keras legacy rules, momentum 0)
# ------------------------------------------------------------------------------------------------
def _f32_inplace(t: torch.Tensor, name: str) -> torch.Tensor:
  require_cuda(t, name)
  if t.dtype != torch.float32 or not t.is_contiguous():
    raise ValueError(f"{name} must be contiguous float32 (it is updated in place)")
  return t


def _sparse_step_args(what: str, table: torch.Tensor, slots: dict, ids: torch.Tensor, grad_rows: torch.Tensor):
  """The argument rules of every sparse optimizer step: `table` and its `slots` ({name: tensor}, updated in place) are
  contiguous float32 of the table's 2-D shape on its device, and `ids` and `grad_rows` [n, d] live there too.  Returns
  (ids flattened, grad_rows as contiguous float32, n, rows, d)."""
  _f32_inplace(table, "table")
  for name, s in slots.items():
    _f32_inplace(s, name)
  ids = require_cuda(ids, "ids").contiguous().view(-1)
  g = f32c(grad_rows, "grad_rows")
  if table.dim() != 2:
    raise ValueError(f"{what}: table must be 2-D, got {tuple(table.shape)}")
  n = ids.numel(); rows, d = table.shape
  for name, s in slots.items():
    if s.shape != table.shape or s.device != table.device:
      raise ValueError(f"{what}: {name} must be {tuple(table.shape)} on {table.device}, got {tuple(s.shape)} on {s.device}")
  if g.shape != (n, d):
    raise ValueError(f"{what}: grad_rows must be [{n},{d}], got {tuple(g.shape)}")
  if ids.device != table.device or g.device != table.device:
    raise ValueError(f"{what}: ids and grad_rows must live on the table's device")
  return ids, g, n, rows, d


def _dense_step_args(what: str, variables: Sequence[torch.Tensor], grads: Sequence[torch.Tensor], slots: dict):
  """The argument rules of every dense multi-tensor step: `variables`, `grads` and each slot list of `slots` ({name:
  list}) have one entry per variable; variables and slots (updated in place) are contiguous float32; every tensor of a
  variable has its shape; all live on one device.  Returns (the grads as contiguous float32, which must stay alive until
  the call is enqueued, and the entry point's leading arguments: the variable, grad and slot pointer arrays, the numels
  and the count)."""
  lists = {"variables": variables, "grads": grads, **slots}
  nv = len(variables)
  if any(len(l) != nv for l in lists.values()):
    names = list(lists)
    raise ValueError(f"{what}: {', '.join(names[:-1])} and {names[-1]} must have the same length")
  gs = []
  for i, (x, g, *ss) in enumerate(zip(variables, grads, *slots.values())):
    _f32_inplace(x, f"variables[{i}]")
    for name, s in zip(slots, ss):
      _f32_inplace(s, f"{name}[{i}]")
    g = f32c(g, f"grads[{i}]")
    if any(t.device != variables[0].device for t in (x, g, *ss)):
      raise ValueError(f"{what}: every tensor must live on one device")
    if g.shape != x.shape or any(s.shape != x.shape for s in ss):
      raise ValueError(f"{what}: {' / '.join(f'{name}[{i}]' for name in ['grads', *slots])} must have the shape "
                       f"{tuple(x.shape)}")
    gs.append(g)
  arr = lambda ts: (ctypes.c_void_p * nv)(*[t.data_ptr() for t in ts])
  numels = (ctypes.c_int64 * nv)(*[x.numel() for x in variables])
  return gs, (arr(variables), arr(gs), *[arr(s) for s in slots.values()], numels, nv)


def sparse_sgd_(table: torch.Tensor, ids: torch.Tensor, grad_rows: torch.Tensor, lr: float) -> None:
  """table[ids[i]] -= lr * grad_rows[i] for every i, duplicates applied one by one in order of occurrence."""
  ids, g, n, rows, d = _sparse_step_args("sparse_sgd_", table, {}, ids, grad_rows)
  if n == 0:
    return
  ws = workspace(lib().tfrs_sparse_sgd_workspace_bytes(n), table.device, "sgd")
  check(lib().tfrs_sparse_sgd_f32(ptr(table), rows, d, ptr(ids), _ffi.ids_dtype_code(ids), n, ptr(g), float(lr), ptr(ws),
                                  ws.numel(), stream()), "sparse_sgd")


def sgd_dense_(params: Sequence[torch.Tensor], grads: Sequence[torch.Tensor], lr: float) -> None:
  """p -= lr * g for every (p, g), in one multi-tensor launch per batch of variables."""
  gs, arrays = _dense_step_args("sgd_dense_", params, grads, {})
  if gs:
    check(lib().tfrs_sgd_dense_f32(*arrays, float(lr), stream()), "sgd_dense")


# ------------------------------------------------------------------------------------------------
# K2 top-k
# ------------------------------------------------------------------------------------------------
def topk_scan(q: torch.Tensor, corpus: torch.Tensor, k: int, index_offset: int = 0,
              state: Optional[Tuple[torch.Tensor, torch.Tensor]] = None,
              out: Optional[Tuple[torch.Tensor, torch.Tensor]] = None) -> Tuple[torch.Tensor, torch.Tensor]:
  """Exact brute-force top-k (CUDA-core path) with optional carried state. Returns ([Q,k_out] f32, [Q,k_out] i64)."""
  q = f32c(q, "queries"); corpus = f32c(corpus, "candidates")
  if q.dim() != 2 or corpus.dim() != 2 or q.shape[1] != corpus.shape[1]:
    raise ValueError(f"topk_scan: shape mismatch {tuple(q.shape)} vs {tuple(corpus.shape)}")
  Q, d = q.shape; N = corpus.shape[0]
  st_s = st_i = None; st_k = 0
  if state is not None and state[0].shape[1] > 0:
    st_s = f32c(state[0], "state scores"); st_i = require_cuda(state[1], "state idx").to(torch.int64).contiguous()
    st_k = st_s.shape[1]
  k_out = min(k, st_k + N)
  if out is None:
    out_s = torch.empty((Q, k), dtype=torch.float32, device=q.device)
    out_i = torch.empty((Q, k), dtype=torch.int64, device=q.device)
  else:
    out_s, out_i = out  # contiguous [Q, k] f32 / i64 views supplied by the caller
  if Q == 0 or k_out == 0:
    return out_s[:, :0], out_i[:, :0]
  wsb = lib().tfrs_topk_scan_workspace_bytes(Q, N, d, k)
  ws = workspace(wsb, q.device, "scan")
  check(lib().tfrs_topk_scan_f32(ptr(q), Q, ptr(corpus), N, d, k, index_offset, ptr(st_s), ptr(st_i), st_k,
                                 ptr(out_s), ptr(out_i), ptr(ws), ws.numel(), stream()), "topk_scan")
  return out_s[:, :k_out], out_i[:, :k_out]


def tc_corpus(corpus: torch.Tensor) -> torch.Tensor:
  """The fp32 corpus as the tensor-core scan reads it.  Its exact re-scoring loads corpus rows as float4 when d % 4 == 0,
  so a corpus that starts off a 16-byte boundary (a contiguous view with a storage offset, e.g. `flat[1:].view(N, d)`)
  is handed over as an aligned copy; any other corpus is returned as is, without a copy."""
  if corpus.shape[-1] % 4 == 0 and corpus.data_ptr() % 16 != 0:
    return corpus.clone(memory_format=torch.contiguous_format)
  return corpus


def index_build(corpus: torch.Tensor, reuse_slot: Optional[str] = None) -> torch.Tensor:
  """Builds the tensor-core screening image (fp16 GMMA tiles + norm bound) of a corpus.  `reuse_slot` builds it in a
  per-stream scratch buffer instead of a fresh allocation (Streaming's per-chunk images)."""
  corpus = tc_corpus(f32c(corpus, "candidates"))
  N, d = corpus.shape
  nb = lib().tfrs_index_bytes(N, d)
  if nb == 0:
    raise NotImplementedError("tensor-core index not available for this shape")
  buf = torch.empty(nb, dtype=torch.uint8, device=corpus.device) if reuse_slot is None else workspace(nb, corpus.device, reuse_slot)
  check(lib().tfrs_index_build(ptr(corpus), N, d, ptr(buf), nb, stream()), "index_build")
  return buf


def _tc_query_chunks(q: torch.Tensor, N: int, k_ws: int):
  """(lo, hi, workspace) for each run of at most TC_MAX_Q_PER_CALL queries: the tensor-core workspace (bin maxima and
  survivor records) grows with Q, so larger batches run chunk by chunk, each workspace sized for k_ws per query."""
  Q, d = q.shape
  for lo in range(0, Q, TC_MAX_Q_PER_CALL):
    hi = min(Q, lo + TC_MAX_Q_PER_CALL)
    yield lo, hi, workspace(lib().tfrs_topk_tc_workspace_bytes(hi - lo, N, d, k_ws), q.device, "tc")


def topk_tc(q: torch.Tensor, corpus: torch.Tensor, index_buf: torch.Tensor, k: int, index_offset: int = 0,
            out: Optional[Tuple[torch.Tensor, torch.Tensor]] = None) -> Tuple[torch.Tensor, torch.Tensor]:
  """wgmma screening + exact rescoring; bit-identical to topk_scan."""
  q = f32c(q, "queries"); corpus = tc_corpus(f32c(corpus, "candidates"))
  Q, d = q.shape; N = corpus.shape[0]
  if out is None:
    out_s = torch.empty((Q, k), dtype=torch.float32, device=q.device)
    out_i = torch.empty((Q, k), dtype=torch.int64, device=q.device)
  else:
    out_s, out_i = out
  for lo, hi, ws in _tc_query_chunks(q, N, k):
    check(lib().tfrs_topk_tc_f32(ptr(q[lo:hi]), hi - lo, ptr(corpus), ptr(index_buf), N, d, k, index_offset, ptr(out_s[lo:hi]),
                                 ptr(out_i[lo:hi]), ptr(ws), ws.numel(), stream()), "topk_tc")
  return out_s, out_i


def tc_supported(Q: int, N: int, d: int, k: int) -> bool:
  """True when (Q, N, d, k) is inside the tensor-core kernels' range (d <= 128, k <= TC_MAX_K, N >= ~256*k)."""
  return lib().tfrs_topk_tc_workspace_bytes(Q, N, d, k) > 0


def uses_tc_scan(Q: int, N: int, d: int, k: int) -> bool:
  """True when a top-k of Q queries over an N x d corpus takes the tensor-core scan.  TC_MIN_N is this module's policy,
  not the kernels': smaller corpora take the exact scan even inside the kernels' range."""
  return N >= TC_MIN_N and tc_supported(Q, N, d, k)


def topk(q: torch.Tensor, corpus: torch.Tensor, k: int, image=None, index_offset: int = 0,
         state: Optional[Tuple[torch.Tensor, torch.Tensor]] = None,
         out: Optional[Tuple[torch.Tensor, torch.Tensor]] = None) -> Tuple[torch.Tensor, torch.Tensor]:
  """Exact top-k of the corpus rows, numbered from index_offset, merged with the carried `state` ([Q, w] scores and
  indices): scores descending, ties -> lower index.  `image` is the corpus's tensor-core image (index_build), the name
  of a scratch slot to build it in, or None.  With an image, uses_tc_scan(Q, N, d, k) and a state of width 0 or k,
  the tensor-core scan runs (a k-wide state is merged in by the sorted-list merge); otherwise topk_scan does."""
  N, d = corpus.shape
  st_k = 0 if state is None else state[0].shape[1]
  if image is None or st_k not in (0, k) or not uses_tc_scan(q.shape[0], N, d, k):
    return topk_scan(q, corpus, k, index_offset=index_offset, state=state, out=out)
  corpus = tc_corpus(f32c(corpus, "candidates"))   # one aligned copy for the image and the scan, if one is needed
  if isinstance(image, str):
    image = index_build(corpus, reuse_slot=image)
  s, i = topk_tc(q, corpus, image, k, index_offset=index_offset, out=out)
  if st_k == 0:
    return s, i
  return topk_merge(torch.stack([state[0], s]), torch.stack([state[1], i]), k, sorted_lists=True)


def _i64(t, name: str, device) -> torch.Tensor:
  if not isinstance(t, torch.Tensor):
    t = torch.as_tensor(t)
  return t.to(device=device, dtype=torch.int64).contiguous()


def topk_tc_exclude(q: torch.Tensor, corpus: torch.Tensor, index_buf: torch.Tensor, k: int, exclusions: torch.Tensor,
                    identifiers: Optional[torch.Tensor] = None, index_offset: int = 0) -> Tuple[torch.Tensor, torch.Tensor]:
  """`query_with_exclusions` fused into the tensor-core scan's finalize step: ([Q,k] f32 original scores,
  [Q,k] i64 global indices).  `identifiers` (integer tensor covering the corpus, or None = the row index) and
  `exclusions` [Q,E] are compared as int64."""
  q = f32c(q, "queries"); corpus = tc_corpus(f32c(corpus, "candidates"))
  Q, d = q.shape; N = corpus.shape[0]
  ex = _i64(exclusions, "exclusions", q.device)
  E = int(ex.shape[1])
  ids = None if identifiers is None else _i64(identifiers, "identifiers", q.device)
  out_s = torch.empty((Q, k), dtype=torch.float32, device=q.device)
  out_i = torch.empty((Q, k), dtype=torch.int64, device=q.device)
  for lo, hi, ws in _tc_query_chunks(q, N, k + E):
    check(lib().tfrs_topk_tc_exclude_f32(ptr(q[lo:hi]), hi - lo, ptr(corpus), ptr(index_buf), N, d, k, index_offset, ptr(ids),
                                         ptr(ex[lo:hi]), E, ptr(out_s[lo:hi]), ptr(out_i[lo:hi]), ptr(ws), ws.numel(), stream()),
          "topk_tc_exclude")
  return out_s, out_i


def topk_tc_count(q: torch.Tensor, corpus: torch.Tensor, index_buf: torch.Tensor, k: int, positive_scores: torch.Tensor
                  ) -> torch.Tensor:
  """min(k, #{candidates scoring strictly above the positive}) per query, int32 [Q] -- the fused score branch of
  FactorizedTopK (no top-K list is produced)."""
  q = f32c(q, "queries"); corpus = tc_corpus(f32c(corpus, "candidates"))
  pos = f32c(positive_scores, "positive_scores").view(-1)
  Q, d = q.shape; N = corpus.shape[0]
  out = torch.empty((Q,), dtype=torch.int32, device=q.device)
  for lo, hi, ws in _tc_query_chunks(q, N, k):
    check(lib().tfrs_topk_tc_count_f32(ptr(q[lo:hi]), hi - lo, ptr(corpus), ptr(index_buf), N, d, k, ptr(pos[lo:hi]),
                                       ptr(out[lo:hi]), ptr(ws), ws.numel(), stream()), "topk_tc_count")
  return out


def exclude_rerank(scores: torch.Tensor, idx: torch.Tensor, exclusions: torch.Tensor, k: int,
                   identifiers: Optional[torch.Tensor] = None) -> Tuple[torch.Tensor, torch.Tensor]:
  """`_exclude` (factorized_top_k.py:83-115) on a fetched [Q, kf] list of (score, global index): returns the original
  scores / indices of the min(k, kf) best after lowering excluded identifiers by 1e5."""
  scores = f32c(scores, "scores"); idx = _i64(idx, "idx", scores.device)
  Q, kf = scores.shape
  ex = _i64(exclusions, "exclusions", scores.device)
  ids = None if identifiers is None else _i64(identifiers, "identifiers", scores.device)
  k_out = min(k, kf)
  out_s = torch.empty((Q, k_out), dtype=torch.float32, device=scores.device)
  out_i = torch.empty((Q, k_out), dtype=torch.int64, device=scores.device)
  if Q and k_out:
    check(lib().tfrs_topk_exclude_rerank_f32(ptr(scores), ptr(idx), Q, kf, ptr(ids), ptr(ex), int(ex.shape[1]), k_out,
                                             ptr(out_s), ptr(out_i), stream()), "exclude_rerank")
  return out_s, out_i


def count_above(scores: torch.Tensor, positive_scores: torch.Tensor) -> torch.Tensor:
  """#{t : scores[q, t] > positive[q]}, int32 [Q] (tf.math.in_top_k's count on a retrieved list)."""
  scores = f32c(scores, "scores"); pos = f32c(positive_scores, "positive_scores").view(-1)
  Q, k = scores.shape
  out = torch.empty((Q,), dtype=torch.int32, device=scores.device)
  check(lib().tfrs_count_above_f32(ptr(scores), scores.stride(0), k, ptr(pos), Q, ptr(out), stream()), "count_above")
  return out


def hits_accumulate(count: torch.Tensor, positive_scores: torch.Tensor, sample_weight: Optional[torch.Tensor],
                    ks: Sequence[int], acc: torch.Tensor) -> None:
  """acc[j] += sum_q w_q [count_q < ks[j], positive finite]; acc[len(ks)] += sum_q w_q.  acc: float64 [len(ks)+1] on
  the device; nothing is synchronised."""
  Q = count.numel()
  w = None if sample_weight is None else f32c(sample_weight, "sample_weight").view(-1)
  if w is not None and w.numel() != Q:
    raise ValueError(f"sample_weight must have one entry per query (got {w.numel()}, expected {Q})")
  karr = (ctypes.c_int32 * len(ks))(*[int(x) for x in ks])
  check(lib().tfrs_topk_hits_accumulate(ptr(count), ptr(f32c(positive_scores, "positive_scores").view(-1)), ptr(w), Q, karr,
                                        len(ks), ptr(acc), stream()), "hits_accumulate")


def topk_merge(scores: torch.Tensor, idx: torch.Tensor, k: int, sorted_lists: bool = False) -> Tuple[torch.Tensor, torch.Tensor]:
  """Merge [L,Q,k_in] lists into the best min(k, L*k_in) per query (score desc, index asc).  `sorted_lists`: every list
  is already in that order (what the scans emit), so the merge ranks by binary search instead of sorting."""
  scores = f32c(scores, "scores"); idx = require_cuda(idx, "idx").to(torch.int64).contiguous()
  L, Q, k_in = scores.shape
  k_out = min(k, L * k_in)
  out_s = torch.empty((Q, k_out), dtype=torch.float32, device=scores.device)
  out_i = torch.empty((Q, k_out), dtype=torch.int64, device=scores.device)
  fn = lib().tfrs_topk_merge_sorted_strided if sorted_lists else lib().tfrs_topk_merge_strided
  check(fn(ptr(scores), ptr(idx), Q * k_in, Q * k_in, L, Q, k_in, k_out, ptr(out_s), ptr(out_i), stream()), "topk_merge")
  return out_s, out_i


# ------------------------------------------------------------------------------------------------
# K14 top-k with overridden rows (examples.movielens.evaluate; DESIGN.md §2 pins the rules)
# ------------------------------------------------------------------------------------------------
OVERRIDE_SCORE = np.float32(-1e6)
OVERRIDE_MAX_K = 2048


def _csr(offsets, rows, Q: int, N: int, device, what: str, sorted_unique: bool):
  """Host offsets (int64 NumPy [Q+1]) and device offsets / rows (int64) of per-query row lists, checked on the host."""
  off = np.ascontiguousarray(offsets.detach().cpu().numpy() if isinstance(offsets, torch.Tensor) else offsets, np.int64)
  r = np.ascontiguousarray(rows.detach().cpu().numpy() if isinstance(rows, torch.Tensor) else rows, np.int64).reshape(-1)
  if off.shape != (Q + 1,) or off[0] != 0 or off[-1] != r.shape[0] or (np.diff(off) < 0).any():
    raise ValueError(f"{what}: offsets must be [Q+1] = [{Q + 1}] non-decreasing from 0 to len(rows) = {r.shape[0]}")
  if r.size and (r.min() < 0 or r.max() >= N):
    raise ValueError(f"{what}: rows must lie in [0, {N})")
  if sorted_unique and r.size > 1:
    ok = np.diff(r) > 0
    starts = off[1:-1]
    ok[starts[(starts > 0) & (starts < r.shape[0])] - 1] = True   # a new list may start lower
    if not ok.all():
      raise ValueError(f"{what}: every query's rows must be sorted and unique")
  return off, torch.from_numpy(off).to(device), torch.from_numpy(r).to(device)


def _override_out(q: torch.Tensor, corpus: torch.Tensor, k: int, what: str):
  q = f32c(q, "queries"); corpus = f32c(corpus, "candidates")
  if q.dim() != 2 or corpus.dim() != 2 or q.shape[1] != corpus.shape[1]:
    raise ValueError(f"{what}: shape mismatch {tuple(q.shape)} vs {tuple(corpus.shape)}")
  if not 0 < k <= OVERRIDE_MAX_K:
    raise ValueError(f"{what}: k={k} out of range (1..{OVERRIDE_MAX_K})")
  k_out = min(k, corpus.shape[0])
  out_s = torch.empty((q.shape[0], k_out), dtype=torch.float32, device=q.device)
  out_i = torch.empty((q.shape[0], k_out), dtype=torch.int64, device=q.device)
  return q, corpus, out_s, out_i


def _overriding_dense(q, corpus, k, off_d, rows_d, users, out_s, out_i, max_chunk_bytes) -> None:
  n = q.shape[0] if users is None else users.numel()
  (_, d), N = q.shape, corpus.shape[0]
  if n == 0 or out_s.shape[1] == 0:
    return
  nb = lib().tfrs_topk_overriding_dense_workspace_bytes(n, N, d, k)
  if max_chunk_bytes is not None:
    nb = min(nb, int(max_chunk_bytes))
  ws = workspace(nb, q.device, "override")
  check(lib().tfrs_topk_overriding_dense_f32(ptr(q), ptr(users), n, ptr(corpus), N, d, k, ptr(off_d), ptr(rows_d), ptr(out_s),
                                             ptr(out_i), out_s.shape[1], ptr(ws), nb, stream()), "topk_overriding_dense")


def topk_overriding_dense(q: torch.Tensor, corpus: torch.Tensor, k: int, offsets, rows,
                          max_chunk_bytes: Optional[int] = None) -> Tuple[torch.Tensor, torch.Tensor]:
  """`topk_overriding` on its dense route for every query: exact scores of a chunk of queries, the listed entries set to
  -1e6, then a per-row selection.  `max_chunk_bytes` caps the workspace of one chunk (default: at most 256 MB)."""
  q, corpus, out_s, out_i = _override_out(q, corpus, k, "topk_overriding_dense")
  _, off_d, rows_d = _csr(offsets, rows, q.shape[0], corpus.shape[0], q.device, "topk_overriding_dense", True)
  _overriding_dense(q, corpus, k, off_d, rows_d, None, out_s, out_i, max_chunk_bytes)
  return out_s, out_i


def override_width(k: int, list_lengths: np.ndarray, N: int) -> np.ndarray:
  """Width of the top-w list each query's scan route reads: min(N, k + e) rounded up to a power of two (at least k, at
  most TC_MAX_K), so the queries fall into a few width classes.  0 marks a query for the dense route."""
  need = np.minimum(N, k + np.asarray(list_lengths, np.int64))
  w = np.maximum(k, 1 << np.ceil(np.log2(np.maximum(need, 1))).astype(np.int64))
  w = np.minimum(np.minimum(w, TC_MAX_K), N)
  return np.where(need <= TC_MAX_K, w, 0)


def topk_overriding(q: torch.Tensor, corpus: torch.Tensor, k: int, offsets, rows, image=None
                    ) -> Tuple[torch.Tensor, torch.Tensor]:
  """Exact top-k of each query over the corpus rows where query u's listed rows rows[offsets[u]:offsets[u+1]] (sorted,
  unique, any length 0..N) score exactly -1e6 instead of their canonical dot.  Order = (score desc, row asc).
  Returns ([Q, min(k, N)] f32 scores, [Q, min(k, N)] i64 rows).

  A query with min(N, k + e) <= TC_MAX_K (e = its list length) takes the scan route: `topk` at its width class
  (`override_width`; the tensor-core scan when `uses_tc_scan` holds and an `image` is given, the exact scan otherwise),
  then one merge kernel drops the listed rows and merges the first k survivors with them.  The top w by true score hold
  at least k survivors, and any survivor outside them ranks after the k-th, so this is exact.  Other queries take
  `topk_overriding_dense`'s route; both routes give the same bits.  `image` is the corpus's tensor-core image
  (index_build), the name of a scratch slot to build it in once, or None.  `offsets` are read on the host."""
  q, corpus, out_s, out_i = _override_out(q, corpus, k, "topk_overriding")
  (Q, d), N = q.shape, corpus.shape[0]
  off_h, off_d, rows_d = _csr(offsets, rows, Q, N, q.device, "topk_overriding", True)
  k_out = out_s.shape[1]
  if Q == 0 or k_out == 0:
    return out_s, out_i
  width = override_width(k, np.diff(off_h), N)
  if image is not None:
    corpus = tc_corpus(corpus)   # one aligned copy for the image and every width class, if one is needed
  if isinstance(image, str) and any(uses_tc_scan(Q, N, d, int(w)) for w in np.unique(width) if w):
    image = index_build(corpus, reuse_slot=image)
  for w in np.unique(width[width > 0]).tolist():
    users = torch.from_numpy(np.nonzero(width == w)[0]).to(q.device)
    ls, li = topk(q.index_select(0, users), corpus, w, image=image)
    check(lib().tfrs_topk_override_merge_f32(ptr(ls), ptr(li), users.numel(), ls.shape[1], ptr(users), ptr(off_d), ptr(rows_d),
                                             k, k_out, ptr(out_s), ptr(out_i), k_out, stream()), "topk_override_merge")
  dense = np.nonzero(width == 0)[0]
  if dense.size:
    _overriding_dense(q, corpus, k, off_d, rows_d, torch.from_numpy(dense).to(q.device), out_s, out_i, None)
  return out_s, out_i


def count_listed(top_rows: torch.Tensor, offsets, rows) -> torch.Tensor:
  """int32 [Q]: per query, how many of its listed rows rows[offsets[u]:offsets[u+1]] (duplicates counted each time)
  appear among top_rows[u] ([Q, kk] int64, kk <= 2048)."""
  top = require_cuda(top_rows, "top_rows").to(torch.int64).contiguous()
  Q, kk = top.shape
  if kk > OVERRIDE_MAX_K:
    raise ValueError(f"count_listed: {kk} rows per query, at most {OVERRIDE_MAX_K}")
  _, off_d, rows_d = _csr(offsets, rows, Q, np.iinfo(np.int64).max, top.device, "count_listed", False)
  out = torch.empty((Q,), dtype=torch.int32, device=top.device)
  check(lib().tfrs_count_listed(ptr(top), Q, kk, kk, ptr(off_d), ptr(rows_d), ptr(out), stream()), "count_listed")
  return out


# ------------------------------------------------------------------------------------------------
# K9 tree-AH: index build and search (DESIGN.md §2 pins every rule)
# ------------------------------------------------------------------------------------------------
TREE_AH_MAX_TRAIN = 100000
TREE_AH_CODEBOOK_ITERATIONS = 10
TREE_AH_MAX_ROWS = 1 << 24
TREE_AH_MAX_K = 2048         # probes, k and k' per query


def tree_ah_assign(x: torch.Tensor, centers: torch.Tensor) -> torch.Tensor:
  """Nearest center by squared L2 (top-1 of [x, 1] . [c, -0.5|c|^2], ties -> lower center) -> int64 [n]."""
  n, d = x.shape
  L = centers.shape[0]
  leaf = torch.empty((n,), dtype=torch.int64, device=x.device)
  ws = workspace(lib().tfrs_tree_ah_assign_workspace_bytes(n, d, L), x.device, "tree_ah")
  check(lib().tfrs_tree_ah_assign_f32(ptr(x), n, d, ptr(centers), L, ptr(leaf), ptr(ws), ws.numel(), stream()), "tree_ah_assign")
  return leaf


def tree_ah_group(leaf: torch.Tensor, L: int) -> Tuple[torch.Tensor, torch.Tensor]:
  """Positions grouped by leaf (ascending leaf, then position) -> (order int32 [n], offsets int32 [L+1])."""
  n = leaf.shape[0]
  order = torch.empty((n,), dtype=torch.int32, device=leaf.device)
  offsets = torch.empty((L + 1,), dtype=torch.int32, device=leaf.device)
  ws = workspace(lib().tfrs_tree_ah_group_workspace_bytes(n), leaf.device, "tree_ah")
  check(lib().tfrs_tree_ah_group(ptr(leaf), n, L, ptr(offsets), ptr(order), ptr(ws), ws.numel(), stream()), "tree_ah_group")
  return order, offsets


def tree_ah_encode(x: torch.Tensor, rows: Optional[torch.Tensor], leaf: torch.Tensor, centroids: torch.Tensor,
                   codebooks: torch.Tensor, dpb: int) -> torch.Tensor:
  """Packed 4-bit residual codes (int32 words [n, W]) of positions p (row = rows[p], or p)."""
  d = x.shape[1]
  n = rows.shape[0] if rows is not None else x.shape[0]
  W = (-(-d // dpb) + 7) // 8
  codes = torch.empty((n, W), dtype=torch.int32, device=x.device)
  check(lib().tfrs_tree_ah_encode(ptr(x), d, ptr(rows), n, ptr(leaf), ptr(centroids), ptr(codebooks), dpb, ptr(codes),
                                  stream()), "tree_ah_encode")
  return codes


def tree_ah_build(candidates: torch.Tensor, num_leaves: int, training_iterations: int, dpb: int) -> dict:
  """Trains the tree and the codebooks and encodes every row (DESIGN.md §2, index build).  Returns the index tensors:
  centroids [L, d], leaf_offsets int32 [L+1], order int32 [N] (row ids, leaf-major), codebooks [B, 16, dpb] and
  codes int32 [N, W] in `order`."""
  import numpy as np
  x = f32c(candidates, "candidates")
  N, d = x.shape
  dev = x.device
  n_train = min(N, TREE_AH_MAX_TRAIN)
  L = min(num_leaves, n_train)
  B = -(-d // dpb)
  perm = np.random.default_rng(0).permutation(N)
  train_rows = np.sort(perm[:n_train])   # ascending row order: the order of every float64 sum
  xt = gather([x], [torch.from_numpy(train_rows).to(dev)])
  cent = gather([x], [torch.from_numpy(perm[:L]).to(dev)])
  for _ in range(training_iterations):
    order_t, off_t = tree_ah_group(tree_ah_assign(xt, cent), L)
    check(lib().tfrs_tree_ah_update_centroids_f32(ptr(xt), d, ptr(order_t), ptr(off_t), L, ptr(cent), stream()),
          "tree_ah_update_centroids")
  leaf_all = tree_ah_assign(x, cent)
  order, offsets = tree_ah_group(leaf_all, L)
  leaf_t = tree_ah_assign(xt, cent)
  pos = torch.from_numpy(np.searchsorted(train_rows, perm[np.arange(16) % n_train]).astype(np.int64)).to(dev)
  cb = torch.empty((B, 16, dpb), dtype=torch.float32, device=dev)
  check(lib().tfrs_tree_ah_init_codebooks_f32(ptr(xt), d, ptr(pos), ptr(leaf_t), ptr(cent), dpb, ptr(cb), stream()),
        "tree_ah_init_codebooks")
  for _ in range(TREE_AH_CODEBOOK_ITERATIONS):
    codes_t = tree_ah_encode(xt, None, leaf_t, cent, cb, dpb)
    check(lib().tfrs_tree_ah_update_codebooks_f32(ptr(xt), d, n_train, ptr(leaf_t), ptr(cent), ptr(codes_t), dpb, ptr(cb),
                                                  stream()), "tree_ah_update_codebooks")
  codes = tree_ah_encode(x, order, leaf_all, cent, cb, dpb)
  return {"centroids": cent, "leaf_offsets": offsets, "order": order, "codebooks": cb, "codes": codes}


def tree_ah_search(q: torch.Tensor, index: dict, rows: Optional[torch.Tensor], num_probes: int, k: int,
                   k_pre: int) -> Tuple[torch.Tensor, torch.Tensor]:
  """Probe, AH-score and pre-select k_pre rows per query, then rescore them exactly when `rows` is given -> top k
  ([Q, k] f32 scores, [Q, k] int64 row ids; (NaN, 0) where the probed leaves hold fewer than k rows).  The sizes
  (d, dimensions per block, L, N) come from the index tensors themselves, which are checked against each other and
  against the queries: the kernels read every buffer with them."""
  q = f32c(q, "queries")
  if q.dim() != 2:
    raise ValueError(f"tree_ah_search: queries must be [Q, d], got {tuple(q.shape)}")
  Q, d = q.shape
  cent, off, order = index["centroids"], index["leaf_offsets"], index["order"]
  cb, codes = index["codebooks"], index["codes"]
  for name, t, dt in (("centroids", cent, torch.float32), ("leaf_offsets", off, torch.int32), ("order", order, torch.int32),
                      ("codebooks", cb, torch.float32), ("codes", codes, torch.int32)):
    require_cuda(t, name)
    if t.dtype != dt or not t.is_contiguous() or t.device != q.device:
      raise ValueError(f"tree_ah_search: index tensor {name} must be a contiguous {dt} tensor on {q.device}")
  if cent.dim() != 2 or cent.shape[1] != d:
    raise ValueError(f"tree_ah_search: queries have d={d} but the index was built for d={cent.shape[1]}")
  L, N = cent.shape[0], order.shape[0]
  dpb = cb.shape[2] if cb.dim() == 3 else 0
  B = -(-d // dpb) if dpb > 0 else 0
  if (dpb < 1 or tuple(cb.shape) != (B, 16, dpb) or tuple(off.shape) != (L + 1,) or order.dim() != 1 or
      tuple(codes.shape) != (N, (B + 7) // 8)):
    raise ValueError("tree_ah_search: inconsistent index tensors "
                     f"(centroids {tuple(cent.shape)}, leaf_offsets {tuple(off.shape)}, order {tuple(order.shape)}, "
                     f"codebooks {tuple(cb.shape)}, codes {tuple(codes.shape)})")
  if rows is not None:
    rows = f32c(rows, "rows")
    if tuple(rows.shape) != (N, d) or rows.device != q.device:
      raise ValueError(f"tree_ah_search: reordering rows must be [{N}, {d}] on {q.device}, got {tuple(rows.shape)}")
  P = min(num_probes, L)
  out_s = torch.empty((Q, k), dtype=torch.float32, device=q.device)
  out_i = torch.empty((Q, k), dtype=torch.int64, device=q.device)
  wsb = lib().tfrs_tree_ah_search_workspace_bytes(Q, d, L, P, dpb, k, k_pre, 1 if rows is not None else 0, N)
  ws = workspace(wsb, q.device, "tree_ah")
  check(lib().tfrs_tree_ah_search_f32(ptr(q), Q, d, ptr(cent), L, ptr(off), ptr(cb), dpb, ptr(codes), ptr(order), N,
                                      ptr(rows), P, k, k_pre, ptr(out_s), ptr(out_i), ptr(ws), ws.numel(), stream()),
        "tree_ah_search")
  return out_s, out_i


def topk_sharded(comm, q: torch.Tensor, corpus_local: torch.Tensor, index_buf: Optional[torch.Tensor], k: int,
                 index_offset: int) -> Tuple[torch.Tensor, torch.Tensor]:
  """The row-sharded BruteForce call through the C ABI: local scan -> one NCCL all-gather -> merge, on every rank."""
  q = f32c(q, "queries"); corpus_local = tc_corpus(f32c(corpus_local, "candidates"))
  Q, d = q.shape; N = corpus_local.shape[0]
  out_s = torch.empty((Q, k), dtype=torch.float32, device=q.device)
  out_i = torch.empty((Q, k), dtype=torch.int64, device=q.device)
  comm.ensure_p2p(Q, k)
  wsb = lib().tfrs_topk_sharded_workspace_bytes(comm.world, Q, N, d, k)
  ws = workspace(wsb + 1024, q.device, "sharded")
  check(lib().tfrs_topk_sharded_f32(comm.handle, ptr(q), Q, ptr(corpus_local), ptr(index_buf), N, d, k, index_offset,
                                    ptr(out_s), ptr(out_i), ptr(ws), ws.numel(), stream()), "topk_sharded")
  return out_s, out_i


def topk_merge_packed(gathered: torch.Tensor, n_lists: int, Q: int, k_in: int, k: int, idx_byte_offset: int,
                      block_bytes: int, sorted_lists: bool = True) -> Tuple[torch.Tensor, torch.Tensor]:
  """Merge the receive buffer of the sharded scan's single all-gather: `n_lists` blocks of `block_bytes`, each
  [scores f32 [Q,k_in] | pad | indices i64 [Q,k_in] at idx_byte_offset].  `sorted_lists` (what the scans emit:
  every list in (score desc, index asc) order) selects the rank-by-binary-search merge instead of the sort."""
  k_out = min(k, n_lists * k_in)
  out_s = torch.empty((Q, k_out), dtype=torch.float32, device=gathered.device)
  out_i = torch.empty((Q, k_out), dtype=torch.int64, device=gathered.device)
  base = gathered.data_ptr()
  fn = lib().tfrs_topk_merge_sorted_strided if sorted_lists else lib().tfrs_topk_merge_strided
  check(fn(ctypes.c_void_p(base), ctypes.c_void_p(base + idx_byte_offset), block_bytes // 4, block_bytes // 8, n_lists, Q,
           k_in, k_out, ptr(out_s), ptr(out_i), stream()), "topk_merge_strided")
  return out_s, out_i


def tc_last_call_stats(Q: int, N: int, d: int, k: int, device=None) -> dict:
  """Survivor / fallback statistics of the most recent topk_tc call with this shape (reads the cached
  workspace; synchronises).  Used by tests to prove the tensor-core path -- not the exact fallback --
  produced the result."""
  out = (ctypes.c_int64 * 10)()
  check(lib().tfrs_topk_tc_layout(Q, N, d, k, out), "topk_tc_layout")
  o_count, o_ovf, o_thr, o_cand, parts, cap, Qp, o_cut = [int(x) for x in out[:8]]
  dev = device if device is not None else torch.device("cuda", torch.cuda.current_device())
  ws = workspace(0, dev, "tc")
  base = (-ws.data_ptr()) % 16
  torch.cuda.synchronize()
  counts = ws[base + o_count: base + o_count + Qp * parts * 4].view(torch.int32).view(Qp, parts)[:Q]
  ovf = ws[base + o_ovf: base + o_ovf + Q * 4].view(torch.int32)
  per_query = counts.sum(1)
  return {"fallback_queries": int((ovf != 0).sum()), "survivors_mean": float(per_query.float().mean()),
          "survivors_max": int(per_query.max()), "parts": parts, "cap_part": cap,
          "part_max": int(counts.max())}


def profile_enable(on: bool) -> None:
  check(lib().tfrs_profile_enable(int(on)), "profile_enable")


def profile_read():
  """-> (stage_ms[4], calls): prep, sample+threshold, filter, finalize; synchronises the device."""
  ms = (ctypes.c_float * 4)(); calls = ctypes.c_int(0)
  check(lib().tfrs_profile_read(ms, ctypes.byref(calls)), "profile_read")
  return [float(x) for x in ms], int(calls.value)


# ------------------------------------------------------------------------------------------------
# exact matmul / scores (autograd-aware)
# ------------------------------------------------------------------------------------------------
def sgemm(a: torch.Tensor, b: torch.Tensor, trans_a: bool = False, trans_b: bool = False,
          out: Optional[torch.Tensor] = None, accumulate: bool = False) -> torch.Tensor:
  a = f32c(a, "a"); b = f32c(b, "b")
  M, K = (a.shape[1], a.shape[0]) if trans_a else (a.shape[0], a.shape[1])
  Kb, N = (b.shape[1], b.shape[0]) if trans_b else (b.shape[0], b.shape[1])
  if K != Kb:
    raise ValueError(f"sgemm: inner dimensions differ ({K} vs {Kb})")
  if out is None:
    out = torch.empty((M, N), dtype=torch.float32, device=a.device)
  check(lib().tfrs_sgemm_f32(int(trans_a), int(trans_b), M, N, K, ptr(a), a.stride(0), ptr(b), b.stride(0),
                             ptr(out), out.stride(0), int(accumulate), stream()), "sgemm")
  return out


class _Scores(torch.autograd.Function):
  """`_compute_score` = matmul(q, c^T) (layers/factorized_top_k.py:320-333) with exact backward."""

  @staticmethod
  def forward(ctx, q, c):
    q = f32c(q, "queries"); c = f32c(c, "candidates")
    ctx.save_for_backward(q, c)
    return sgemm(q, c, False, True)

  @staticmethod
  def backward(ctx, g):
    q, c = ctx.saved_tensors
    g = f32c(g, "grad")
    dq = sgemm(g, c, False, False) if ctx.needs_input_grad[0] else None
    dc = sgemm(g, q, True, False) if ctx.needs_input_grad[1] else None
    return dq, dc


def scores(q: torch.Tensor, c: torch.Tensor) -> torch.Tensor:
  return _Scores.apply(q, c)


class _Matmul(torch.autograd.Function):
  """x @ w with our exact SGEMM (used by the low-rank Cross path)."""

  @staticmethod
  def forward(ctx, x, w):
    x = f32c(x, "x"); w = f32c(w, "w")
    ctx.save_for_backward(x, w)
    return sgemm(x, w, False, False)

  @staticmethod
  def backward(ctx, g):
    x, w = ctx.saved_tensors
    g = f32c(g, "grad")
    dx = sgemm(g, w, False, True) if ctx.needs_input_grad[0] else None
    dw = sgemm(x, g, True, False) if ctx.needs_input_grad[1] else None
    return dx, dw


def matmul(x: torch.Tensor, w: torch.Tensor) -> torch.Tensor:
  return _Matmul.apply(x, w)


def rowwise_dot(a: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
  a = f32c(a, "a"); b = f32c(b, "b")
  out = torch.empty((a.shape[0],), dtype=torch.float32, device=a.device)
  check(lib().tfrs_rowwise_dot_f32(ptr(a), ptr(b), a.shape[0], a.shape[1], ptr(out), stream()), "rowwise_dot")
  return out


# ------------------------------------------------------------------------------------------------
# K3 in-batch softmax loss
# ------------------------------------------------------------------------------------------------
SOFTMAX_TC_MIN_B = 512  # below this the exact CUDA-core forward is launch-latency bound anyway


def inbatch_softmax_tc(q: torch.Tensor, c: torch.Tensor, sample_weight: Optional[torch.Tensor] = None,
                       inv_temperature: float = 1.0, candidate_bias: Optional[torch.Tensor] = None,
                       candidate_ids: Optional[torch.Tensor] = None, score_mask: Optional[torch.Tensor] = None):
  """Tensor-core forward only (any B): returns (loss scalar, lse [B]).  Raises NotImplementedError when d > 128.
  `candidate_bias` [C] is added to every logit of its column (after the temperature); `candidate_ids` (int64 [C]) removes
  accidental hits and `score_mask` (uint8 [B, C], nonzero = keep) masks logits, as in inbatch_softmax_loss."""
  q = f32c(q, "query_embeddings"); c = f32c(c, "candidate_embeddings")
  B, d = q.shape; C = c.shape[0]
  w = None if sample_weight is None else f32c(sample_weight, "sample_weight").view(-1)
  loss = torch.empty((1,), dtype=torch.float32, device=q.device)
  lse = torch.empty((B,), dtype=torch.float32, device=q.device)
  cb = None if candidate_bias is None else f32c(candidate_bias, "candidate_bias").view(-1)
  wsb = lib().tfrs_inbatch_softmax_tc_workspace_bytes(B, C, d, int(candidate_ids is not None), int(score_mask is not None))
  ws = workspace(wsb, q.device, "softmax_tc")
  check(lib().tfrs_inbatch_softmax_tc_fwd(ptr(q), ptr(c), B, C, d, c_f(inv_temperature), ptr(w), ptr(cb), ptr(candidate_ids),
                                          ptr(score_mask), ptr(loss), ptr(lse), ptr(ws), ws.numel(), stream()),
        "inbatch_softmax_tc_fwd")
  return loss.view(()), lse


def _ids_i64(candidate_ids, C: int, device) -> torch.Tensor:
  """candidate ids of any type -> int64 [C] on the device.  Integer tensors are used as they are; anything else (strings,
  NumPy object arrays, float ids) is factorised on the host -- only EQUALITY of ids matters to accidental-hit removal."""
  if isinstance(candidate_ids, torch.Tensor) and not candidate_ids.dtype.is_floating_point and candidate_ids.dtype != torch.bool:
    t = candidate_ids.reshape(-1).to(device=device, dtype=torch.int64).contiguous()
  else:
    import numpy as np
    arr = candidate_ids.detach().cpu().numpy() if isinstance(candidate_ids, torch.Tensor) else np.asarray(candidate_ids)
    _, inv = np.unique(arr.reshape(-1), return_inverse=True)
    t = torch.as_tensor(inv.astype(np.int64), device=device)
  if t.numel() != C:
    raise ValueError(f"candidate_ids must have one entry per candidate (got {t.numel()}, expected {C})")
  return t


class _InBatchSoftmax(torch.autograd.Function):

  @staticmethod
  def forward(ctx, q, c, sample_weight, inv_temperature, candidate_bias=None, candidate_ids=None, score_mask=None):
    q = f32c(q, "query_embeddings"); c = f32c(c, "candidate_embeddings")
    B, d = q.shape; C = c.shape[0]
    w = None if sample_weight is None else f32c(sample_weight, "sample_weight").view(-1)
    cb = None if candidate_bias is None else f32c(candidate_bias, "candidate_bias").view(-1)
    if cb is not None and cb.numel() != C:
      raise ValueError(f"candidate_bias must have one entry per candidate (got {cb.numel()}, expected {C})")
    if w is not None and w.numel() != B:
      raise ValueError(f"sample_weight must have one entry per query (got {w.numel()}, expected {B})")
    ids = None if candidate_ids is None else _ids_i64(candidate_ids, C, q.device)
    mask = None
    if score_mask is not None:
      mask = require_cuda(score_mask, "score_mask")
      if tuple(mask.shape) != (B, C):
        raise ValueError(f"score_mask must be [{B},{C}], got {tuple(mask.shape)}")
      mask = (mask if mask.dtype == torch.bool else mask != 0).contiguous().view(torch.uint8)
    ext = ids is not None or mask is not None
    # the tensor-core kernels work in log2 units scaled by 1/T > 0; any other temperature takes the exact path
    if (cb is not None or ext) and not (inv_temperature > 0 and inbatch_softmax_bias_supported(B, C, d)):
      raise NotImplementedError("inbatch_softmax_loss: candidate_bias / candidate_ids / score_mask need the tensor-core path "
                                f"(B >= {SOFTMAX_TC_MIN_B}, d <= 64, temperature > 0); got B={B}, d={d}, "
                                f"1/temperature={inv_temperature}")
    used_tc = inv_temperature > 0 and B >= SOFTMAX_TC_MIN_B and \
        lib().tfrs_inbatch_softmax_tc_workspace_bytes(B, C, d, int(ids is not None), int(mask is not None)) > 0
    if used_tc:  # tensor-core forward (hi/lo fp16 split, fp32 accumulate, online log-sum-exp epilogue)
      loss, lse = inbatch_softmax_tc(q, c, w, inv_temperature, cb, ids, mask)
    else:
      loss = torch.empty((1,), dtype=torch.float32, device=q.device)
      lse = torch.empty((B,), dtype=torch.float32, device=q.device)
      wsb = lib().tfrs_inbatch_softmax_workspace_bytes(B, C, d)
      ws = workspace(wsb, q.device, "softmax")
      check(lib().tfrs_inbatch_softmax_fwd(ptr(q), ptr(c), B, C, d, c_f(inv_temperature), ptr(w), ptr(loss), ptr(lse),
                                           ptr(ws), ws.numel(), stream()), "inbatch_softmax_fwd")
    empty = torch.empty(0, device=q.device)
    ctx.save_for_backward(q, c, lse, w if w is not None else empty, cb if cb is not None else empty,
                          ids if ids is not None else empty, mask if mask is not None else empty)
    ctx.has_w = w is not None
    ctx.has_cb = cb is not None
    ctx.has_ids = ids is not None
    ctx.has_mask = mask is not None
    ctx.inv_t = inv_temperature
    ctx.used_tc = used_tc
    return loss.view(())

  @staticmethod
  def backward(ctx, g):
    q, c, lse, w, cb, ids, mask = ctx.saved_tensors
    B, d = q.shape; C = c.shape[0]
    g = f32c(g, "grad").view(1)
    if ctx.used_tc and lib().tfrs_inbatch_softmax_tc_bwd_workspace_bytes(B, C, d, int(ctx.has_ids), int(ctx.has_mask)):
      # tensor-core backward: same split products as the forward pass that produced `lse`
      dq, dc = inbatch_softmax_tc_bwd(q, c, lse, w if ctx.has_w else None, ctx.inv_t, g, cb if ctx.has_cb else None,
                                      ids if ctx.has_ids else None, mask if ctx.has_mask else None)
      return dq, dc, None, None, None, None, None
    if ctx.has_cb or ctx.has_ids or ctx.has_mask:
      raise NotImplementedError("inbatch_softmax_loss backward with loss options needs the tensor-core path")
    dq = torch.empty_like(q); dc = torch.empty_like(c)
    wsb = lib().tfrs_inbatch_softmax_workspace_bytes(B, C, d)
    ws = workspace(wsb, q.device, "softmax")
    check(lib().tfrs_inbatch_softmax_bwd(ptr(q), ptr(c), B, C, d, c_f(ctx.inv_t), ptr(w) if ctx.has_w else None,
                                         ptr(lse), ptr(g), ptr(dq), ptr(dc), ptr(ws), ws.numel(), stream()),
          "inbatch_softmax_bwd")
    return dq, dc, None, None, None, None, None


def inbatch_softmax_bwd_exact(q, c, lse, sample_weight=None, inv_temperature: float = 1.0, grad_loss=None):
  """Exact fp32 CUDA-core backward for a given saved `lse` (the anchor the tensor-core backward is tested against)."""
  q = f32c(q, "query_embeddings"); c = f32c(c, "candidate_embeddings"); lse = f32c(lse, "lse")
  B, d = q.shape; C = c.shape[0]
  w = None if sample_weight is None else f32c(sample_weight, "sample_weight").view(-1)
  g = None if grad_loss is None else f32c(grad_loss, "grad").view(1)
  dq = torch.empty_like(q); dc = torch.empty_like(c)
  ws = workspace(lib().tfrs_inbatch_softmax_workspace_bytes(B, C, d), q.device, "softmax")
  check(lib().tfrs_inbatch_softmax_bwd(ptr(q), ptr(c), B, C, d, c_f(inv_temperature), ptr(w), ptr(lse), ptr(g), ptr(dq), ptr(dc),
                                       ptr(ws), ws.numel(), stream()), "inbatch_softmax_bwd")
  return dq, dc


def inbatch_softmax_tc_bwd(q, c, lse, sample_weight=None, inv_temperature: float = 1.0, grad_loss=None, candidate_bias=None,
                           candidate_ids: Optional[torch.Tensor] = None, score_mask: Optional[torch.Tensor] = None):
  """Tensor-core backward only (any B, d <= 64): returns (dq, dc) for the given saved `lse`; options as inbatch_softmax_tc."""
  q = f32c(q, "query_embeddings"); c = f32c(c, "candidate_embeddings"); lse = f32c(lse, "lse")
  B, d = q.shape; C = c.shape[0]
  w = None if sample_weight is None else f32c(sample_weight, "sample_weight").view(-1)
  g = None if grad_loss is None else f32c(grad_loss, "grad").view(1)
  dq = torch.empty_like(q); dc = torch.empty_like(c)
  wsb = lib().tfrs_inbatch_softmax_tc_bwd_workspace_bytes(B, C, d, int(candidate_ids is not None), int(score_mask is not None))
  ws = workspace(wsb, q.device, "softmax_tc_bwd")
  cb = None if candidate_bias is None else f32c(candidate_bias, "candidate_bias").view(-1)
  check(lib().tfrs_inbatch_softmax_tc_bwd(ptr(q), ptr(c), B, C, d, c_f(inv_temperature), ptr(w), ptr(cb), ptr(candidate_ids),
                                          ptr(score_mask), ptr(lse), ptr(g), ptr(dq), ptr(dc), ptr(ws), ws.numel(), stream()),
        "inbatch_softmax_tc_bwd")
  return dq, dc


def inbatch_softmax_bias_supported(B: int, C: int, d: int) -> bool:
  """True when the loss with a per-candidate logit bias can run fused (tensor-core forward AND backward)."""
  return (B >= SOFTMAX_TC_MIN_B and lib().tfrs_inbatch_softmax_tc_workspace_bytes(B, C, d, 0, 0) > 0 and
          lib().tfrs_inbatch_softmax_tc_bwd_workspace_bytes(B, C, d, 0, 0) > 0)


def inbatch_softmax_loss(q: torch.Tensor, c: torch.Tensor, sample_weight: Optional[torch.Tensor] = None,
                         temperature: Optional[float] = None, candidate_bias: Optional[torch.Tensor] = None,
                         candidate_ids=None, score_mask: Optional[torch.Tensor] = None) -> torch.Tensor:
  """sum_i w_i * (logsumexp_j(l_ij) - l_ii),  l_ij = q_i.c_j / T + b_j  -- tasks/retrieval.py:178-210;
  b = candidate_bias (e.g. -log(clip(p, 1e-6, 1)): the sampling-probability correction, :190-192), no gradient;
  candidate_ids: accidental-hit removal (:194-200) -- l_ij = MIN_FLOAT where id_j == id_i, j != i;
  score_mask [B,C]: l_ij = MIN_FLOAT where the mask is False (:202-203)."""
  inv_t = 1.0 if temperature is None else 1.0 / float(temperature)
  return _InBatchSoftmax.apply(q, c, sample_weight, inv_t, candidate_bias, candidate_ids, score_mask)


class _MaxSimSoftmax(torch.autograd.Function):
  """In-batch softmax loss on multi-head queries [B,H,d]: scores = max over heads (tasks/retrieval.py:172-176)."""

  @staticmethod
  def forward(ctx, q, c, sample_weight, inv_temperature):
    q = f32c(q, "query_embeddings"); c = f32c(c, "candidate_embeddings")
    B, H, d = q.shape; C = c.shape[0]
    w = None if sample_weight is None else f32c(sample_weight, "sample_weight").view(-1)
    if w is not None and w.numel() != B:
      raise ValueError(f"sample_weight must have one entry per query (got {w.numel()}, expected {B})")
    loss = torch.empty((1,), dtype=torch.float32, device=q.device)
    lse = torch.empty((B,), dtype=torch.float32, device=q.device)
    ws = workspace(lib().tfrs_inbatch_softmax_maxsim_workspace_bytes(B, H, C, d), q.device, "softmax")
    check(lib().tfrs_inbatch_softmax_maxsim_fwd(ptr(q), ptr(c), B, H, C, d, c_f(inv_temperature), ptr(w), ptr(loss), ptr(lse),
                                                ptr(ws), ws.numel(), stream()), "inbatch_softmax_maxsim_fwd")
    ctx.save_for_backward(q, c, lse, w if w is not None else torch.empty(0, device=q.device))
    ctx.has_w = w is not None
    ctx.inv_t = inv_temperature
    return loss.view(())

  @staticmethod
  def backward(ctx, g):
    q, c, lse, w = ctx.saved_tensors
    B, H, d = q.shape; C = c.shape[0]
    g = f32c(g, "grad").view(1)
    dq = torch.empty_like(q); dc = torch.empty_like(c)
    ws = workspace(lib().tfrs_inbatch_softmax_maxsim_workspace_bytes(B, H, C, d), q.device, "softmax")
    check(lib().tfrs_inbatch_softmax_maxsim_bwd(ptr(q), ptr(c), B, H, C, d, c_f(ctx.inv_t), ptr(w) if ctx.has_w else None, ptr(lse),
                                                ptr(g), ptr(dq), ptr(dc), ptr(ws), ws.numel(), stream()), "inbatch_softmax_maxsim_bwd")
    return dq, dc, None, None


def inbatch_softmax_maxsim_loss(q: torch.Tensor, c: torch.Tensor, sample_weight: Optional[torch.Tensor] = None,
                                temperature: Optional[float] = None) -> torch.Tensor:
  """sum_i w_i (logsumexp_j(max_h q_ih.c_j / T) - max_h q_ih.c_i / T) for q [B,H,d] (tasks/retrieval.py:172-210)."""
  inv_t = 1.0 if temperature is None else 1.0 / float(temperature)
  return _MaxSimSoftmax.apply(q, c, sample_weight, inv_t)


# ------------------------------------------------------------------------------------------------
# hard-negative mining loss (top-K scan + sparse softmax)
# ------------------------------------------------------------------------------------------------
def hard_negative_supported(B: int, C: int, d: int, num_hard_negatives: int) -> bool:
  """True when Retrieval(num_hard_negatives=n) can run on the top-K scan instead of the [B,C] logits."""
  return num_hard_negatives >= 1 and C >= B and min(num_hard_negatives + 1, C) <= 2048


class _HardNegativeSoftmax(torch.autograd.Function):

  @staticmethod
  def forward(ctx, q, c, num_hard_negatives, sample_weight, inv_temperature):
    q = f32c(q, "query_embeddings"); c = f32c(c, "candidate_embeddings")
    B = q.shape[0]; C = c.shape[0]
    if not inv_temperature > 0:
      raise NotImplementedError("hard_negative_softmax_loss needs a positive temperature")
    k1 = min(int(num_hard_negatives) + 1, C)
    w = None if sample_weight is None else f32c(sample_weight, "sample_weight").view(-1)
    if w is not None and w.numel() != B:
      raise ValueError(f"sample_weight must have one entry per query (got {w.numel()}, expected {B})")
    qd, cd = q.detach(), c.detach()
    top_s, top_i = topk(qd, cd, k1, image="hardneg_index")
    pos = rowwise_dot(qd, cd[:B])
    loss = torch.empty((1,), dtype=torch.float32, device=q.device)
    coef = torch.empty((B, k1 + 2), dtype=torch.float32, device=q.device)
    check(lib().tfrs_hardneg_loss_fwd(ptr(top_s), ptr(top_i), B, k1, ptr(pos), c_f(inv_temperature), ptr(w), ptr(loss), ptr(coef),
                                      stream()), "hardneg_loss_fwd")
    ctx.save_for_backward(q, c, top_i, coef)
    ctx.k1 = k1
    return loss.view(())

  @staticmethod
  def backward(ctx, g):
    q, c, top_i, coef = ctx.saved_tensors
    B, d = q.shape; C = c.shape[0]
    g = f32c(g, "grad").view(1)
    dq = torch.empty_like(q); dc = torch.empty_like(c)
    check(lib().tfrs_hardneg_loss_bwd(ptr(q), ptr(c), B, C, d, ptr(top_i), ctx.k1, ptr(coef), ptr(g), ptr(dq), ptr(dc), stream()),
          "hardneg_loss_bwd")
    return dq, dc, None, None, None


def hard_negative_softmax_loss(q: torch.Tensor, c: torch.Tensor, num_hard_negatives: int,
                               sample_weight: Optional[torch.Tensor] = None, temperature: Optional[float] = None) -> torch.Tensor:
  """Retrieval loss with HardNegativeMining(n) (tasks/retrieval.py:205-210, layers/loss.py:61-111): softmax cross-entropy
  over the positive and the n highest-scoring other candidates of each query."""
  inv_t = 1.0 if temperature is None else 1.0 / float(temperature)
  return _HardNegativeSoftmax.apply(q, c, int(num_hard_negatives), sample_weight, inv_t)


# ------------------------------------------------------------------------------------------------
# K4 sparse Adagrad
# ------------------------------------------------------------------------------------------------
def sparse_adagrad_(table: torch.Tensor, accum: torch.Tensor, ids: torch.Tensor, grad_rows: torch.Tensor,
                    lr: float, eps: float = 1e-7, eps_inside_sqrt: bool = True) -> None:
  ids, g, n, rows, d = _sparse_step_args("sparse_adagrad_", table, {"accum": accum}, ids, grad_rows)
  ws = workspace(lib().tfrs_sparse_adagrad_workspace_bytes(n, d), table.device, "adagrad")
  check(lib().tfrs_sparse_adagrad_f32(ptr(table), ptr(accum), rows, d, ptr(ids), _ffi.ids_dtype_code(ids), n,
                                      ptr(g), c_f(lr), c_f(eps), int(eps_inside_sqrt), ptr(ws), ws.numel(), stream()),
        "sparse_adagrad")


# ------------------------------------------------------------------------------------------------
# K7 ClippyAdagrad
# ------------------------------------------------------------------------------------------------
def _clippy_flags(clip_accumulator_update: bool, use_standard_accumulator_update: bool) -> int:
  return (1 if clip_accumulator_update else 0) | (2 if use_standard_accumulator_update else 0)


def sparse_clippy_adagrad_(table: torch.Tensor, accum: torch.Tensor, ids: torch.Tensor, grad_rows: torch.Tensor,
                           lr: float, eps: float, variable_relative_threshold: float, accumulator_relative_threshold: float,
                           absolute_threshold: float, clip_accumulator_update: bool = False,
                           use_standard_accumulator_update: bool = False,
                           clipping_factor: Optional[torch.Tensor] = None) -> None:
  """ClippyAdagrad step of one embedding table on the rows `ids` (duplicates summed in order of occurrence).  The
  variable's clipping factor is written to the 0-d float32 device tensor `clipping_factor` when given."""
  ids, g, n, rows, d = _sparse_step_args("sparse_clippy_adagrad_", table, {"accum": accum}, ids, grad_rows)
  if clipping_factor is not None:
    _f32_inplace(clipping_factor, "clipping_factor")
    if clipping_factor.numel() != 1:
      raise ValueError("sparse_clippy_adagrad_: clipping_factor must hold one float")
  wsb = lib().tfrs_sparse_clippy_adagrad_workspace_bytes(n, d)
  ws = workspace(wsb, table.device, "clippy")
  check(lib().tfrs_sparse_clippy_adagrad_f32(
      ptr(table), ptr(accum), rows, d, ptr(ids), _ffi.ids_dtype_code(ids), n, ptr(g), c_f(lr), c_f(eps),
      c_f(variable_relative_threshold), c_f(accumulator_relative_threshold), c_f(absolute_threshold),
      _clippy_flags(clip_accumulator_update, use_standard_accumulator_update), ptr(clipping_factor), ptr(ws), ws.numel(),
      stream()), "sparse_clippy_adagrad")


def clippy_adagrad_dense_(variables: Sequence[torch.Tensor], grads: Sequence[torch.Tensor], accums: Sequence[torch.Tensor],
                          lr: float, eps: float, variable_relative_threshold: float, accumulator_relative_threshold: float,
                          absolute_threshold: float, clip_accumulator_update: bool = False,
                          use_standard_accumulator_update: bool = False,
                          clipping_factors: Optional[torch.Tensor] = None) -> None:
  """ClippyAdagrad step of a list of dense variables in one multi-tensor call (one clipping factor per variable,
  written to the float32 device tensor `clipping_factors` [len(variables)] when given)."""
  gs, arrays = _dense_step_args("clippy_adagrad_dense_", variables, grads, {"accums": accums})
  if not gs:
    return
  nv, dev = len(gs), variables[0].device
  if clipping_factors is not None:
    _f32_inplace(clipping_factors, "clipping_factors")
    if clipping_factors.numel() != nv or clipping_factors.device != dev:
      raise ValueError(f"clippy_adagrad_dense_: clipping_factors must hold {nv} floats on {dev}")
  ws = workspace(lib().tfrs_clippy_adagrad_dense_workspace_bytes(nv), dev, "clippy")
  check(lib().tfrs_clippy_adagrad_dense_f32(
      *arrays, c_f(lr), c_f(eps), c_f(variable_relative_threshold),
      c_f(accumulator_relative_threshold), c_f(absolute_threshold),
      _clippy_flags(clip_accumulator_update, use_standard_accumulator_update), ptr(clipping_factors), ptr(ws), ws.numel(),
      stream()), "clippy_adagrad_dense")


# ------------------------------------------------------------------------------------------------
# K10 Adam
# ------------------------------------------------------------------------------------------------
def adam_alpha(learning_rate: float, beta_1: float, beta_2: float, t: int) -> float:
  """The step size of Adam's step t (1-based): lr * sqrt(1 - beta_2^t) / (1 - beta_1^t), evaluated in float64 from the
  fp32-rounded hyperparameters and rounded once to fp32."""
  lr, b1, b2 = (c_f(x).value for x in (learning_rate, beta_1, beta_2))
  return c_f(lr * math.sqrt(1.0 - b2 ** t) / (1.0 - b1 ** t)).value


def sparse_adam_(table: torch.Tensor, m: torch.Tensor, v: torch.Tensor, ids: torch.Tensor, grad_rows: torch.Tensor,
                 alpha: float, beta_1: float, beta_2: float, epsilon: float, lazy: bool = False) -> None:
  """Adam step of one embedding table whose gradient rows `grad_rows` belong to the rows `ids` (duplicates summed in order
  of occurrence, out-of-range ids skipped).  `alpha` is the step size of `adam_alpha`.  Not lazy: every row of the table
  and of its slots `m` / `v` is updated (the untouched ones decay); lazy: only the touched rows."""
  ids, g, n, rows, d = _sparse_step_args("sparse_adam_", table, {"m": m, "v": v}, ids, grad_rows)
  ws = workspace(lib().tfrs_sparse_adam_workspace_bytes(n, rows), table.device, "adam")
  check(lib().tfrs_sparse_adam_f32(
      ptr(table), ptr(m), ptr(v), rows, d, ptr(ids), _ffi.ids_dtype_code(ids), n, ptr(g), c_f(alpha), c_f(beta_1),
      c_f(beta_2), c_f(epsilon), int(bool(lazy)), ptr(ws), ws.numel(), stream()), "sparse_adam")


def adam_dense_(variables: Sequence[torch.Tensor], grads: Sequence[torch.Tensor], ms: Sequence[torch.Tensor],
                vs: Sequence[torch.Tensor], alpha: float, beta_1: float, beta_2: float, epsilon: float) -> None:
  """Adam step of a list of dense variables and their slots `ms` / `vs` in one multi-tensor call; `alpha` is the step
  size of `adam_alpha`."""
  gs, arrays = _dense_step_args("adam_dense_", variables, grads, {"ms": ms, "vs": vs})
  if gs:
    check(lib().tfrs_adam_dense_f32(*arrays, c_f(alpha), c_f(beta_1), c_f(beta_2), c_f(epsilon), stream()), "adam_dense")


# ------------------------------------------------------------------------------------------------
# K12 FTRL
# ------------------------------------------------------------------------------------------------
def ftrl_l2(l2: float, beta: float, lr: float) -> float:
  """The l2 strength FTRL's kernels take: l2 + beta / (2*lr), evaluated in fp32 one operation at a time from the
  fp32-rounded arguments, as tf-keras folds `beta` into l2 before calling the raw op."""
  l2, beta, lr = (c_f(x).value for x in (l2, beta, lr))
  return c_f(l2 + c_f(beta / c_f(2.0 * lr).value).value).value


def sparse_ftrl_(table: torch.Tensor, accum: torch.Tensor, linear: torch.Tensor, ids: torch.Tensor,
                 grad_rows: torch.Tensor, lr: float, lr_power: float, l1: float, l2a: float,
                 l2_shrinkage: float) -> None:
  """FTRL step of one embedding table whose gradient rows `grad_rows` belong to the rows `ids` (duplicates summed in order
  of occurrence, out-of-range ids skipped).  `l2a` is the l2 strength of `ftrl_l2`.  Only the touched rows of the table
  and of its slots `accum` / `linear` change."""
  ids, g, n, rows, d = _sparse_step_args("sparse_ftrl_", table, {"accum": accum, "linear": linear}, ids, grad_rows)
  ws = workspace(lib().tfrs_sparse_ftrl_workspace_bytes(n), table.device, "ftrl")
  check(lib().tfrs_sparse_ftrl_f32(
      ptr(table), ptr(accum), ptr(linear), rows, d, ptr(ids), _ffi.ids_dtype_code(ids), n, ptr(g), c_f(lr), c_f(lr_power),
      c_f(l1), c_f(l2a), c_f(l2_shrinkage), ptr(ws), ws.numel(), stream()), "sparse_ftrl")


def ftrl_dense_(variables: Sequence[torch.Tensor], grads: Sequence[torch.Tensor], accums: Sequence[torch.Tensor],
                linears: Sequence[torch.Tensor], lr: float, lr_power: float, l1: float, l2a: float,
                l2_shrinkage: float) -> None:
  """FTRL step of a list of dense variables and their slots `accums` / `linears` in one multi-tensor call; `l2a` is the
  l2 strength of `ftrl_l2`."""
  gs, arrays = _dense_step_args("ftrl_dense_", variables, grads, {"accums": accums, "linears": linears})
  if gs:
    check(lib().tfrs_ftrl_dense_f32(*arrays, c_f(lr), c_f(lr_power), c_f(l1), c_f(l2a), c_f(l2_shrinkage), stream()),
          "ftrl_dense")


# ------------------------------------------------------------------------------------------------
# K5 cross
# ------------------------------------------------------------------------------------------------
# Cross layers at least this large run their forward GEMM on the tensor cores (fp16 hi/lo split, fp32 accumulate).
CROSS_TC_MIN_B = 1024
CROSS_TC_MIN_D = 64


class _Cross(torch.autograd.Function):

  @staticmethod
  def forward(ctx, x0, x, W, bias, diag_scale, x_amax):
    x0 = f32c(x0, "x0"); x = f32c(x, "x"); W = f32c(W, "kernel")
    b = None if bias is None else f32c(bias, "bias")
    B, D = x0.shape
    out = torch.empty_like(x0)
    need_grad = any(ctx.needs_input_grad[:4])
    prod = torch.empty_like(x0) if need_grad else None
    ctx.used_tc = B >= CROSS_TC_MIN_B and D >= CROSS_TC_MIN_D and W.shape == (D, D)
    # max |out| as float bits, produced by the tensor-core epilogue: the next layer of a stack uses it as its rescale
    # statistic instead of a pass over its input (0 on the exact path: "unknown")
    out_amax = torch.zeros((1,), dtype=torch.int32, device=x0.device)
    if ctx.used_tc:
      ws = workspace(lib().tfrs_cross_tc_workspace_bytes(B, D), x0.device, "cross_tc")
      check(lib().tfrs_cross_tc_fwd_f32(ptr(x0), ptr(x), ptr(W), ptr(b), B, D, D, c_f(diag_scale), ptr(out), ptr(prod),
                                        ptr(x_amax), ptr(out_amax), ptr(ws), ws.numel(), stream()), "cross_tc_fwd")
    else:
      check(lib().tfrs_cross_fwd_f32(ptr(x0), ptr(x), ptr(W), ptr(b), B, D, D, c_f(diag_scale), ptr(out), ptr(prod),
                                     stream()), "cross_fwd")
    if need_grad:
      ctx.save_for_backward(x0, x, W, prod)
    ctx.diag = diag_scale
    ctx.has_bias = b is not None
    ctx.mark_non_differentiable(out_amax)
    return out, out_amax

  @staticmethod
  def backward(ctx, g, _g_amax=None):
    x0, x, W, prod = ctx.saved_tensors
    g = f32c(g, "grad")
    B, D = x0.shape
    n0, n1, n2, n3 = ctx.needs_input_grad[:4]
    dx0 = torch.empty_like(x0) if n0 else None
    dx = torch.empty_like(x) if n1 else None
    dW = torch.empty_like(W) if n2 else None
    db = torch.empty((D,), dtype=torch.float32, device=x0.device) if (n3 and ctx.has_bias) else None
    if ctx.used_tc:  # the two GEMMs (dx, dW) on the tensor cores
      ws = workspace(lib().tfrs_cross_tc_bwd_workspace_bytes(B, D), x0.device, "cross_tc_bwd")
      check(lib().tfrs_cross_tc_bwd_f32(ptr(x0), ptr(x), ptr(W), ptr(prod), ptr(g), B, D, D, c_f(ctx.diag), ptr(dx0), ptr(dx),
                                        ptr(dW), ptr(db), ptr(ws), ws.numel(), stream()), "cross_tc_bwd")
      return dx0, dx, dW, db, None, None
    wsb = lib().tfrs_cross_bwd_workspace_bytes(B, D)
    ws = workspace(wsb, x0.device, "cross")
    check(lib().tfrs_cross_bwd_f32(ptr(x0), ptr(x), ptr(W), ptr(prod), ptr(g), B, D, D, c_f(ctx.diag), ptr(dx0), ptr(dx),
                                   ptr(dW), ptr(db), ptr(ws), ws.numel(), stream()), "cross_bwd")
    return dx0, dx, dW, db, None, None


def cross(x0: torch.Tensor, x: torch.Tensor, W: torch.Tensor, bias: Optional[torch.Tensor], diag_scale: float = 0.0
          ) -> torch.Tensor:
  """x0 * (x @ W + bias + diag_scale * x) + x   (layers/feature_interaction/dcn.py:176-186).

  Stacked layers (`x = cross(x0, x)`): the output carries max |out| from the kernel's epilogue (`_tfrs_amax`), and a later
  call whose `x` is that very tensor, unmodified, skips its statistics pass over x -- same bits, one HBM pass less."""
  hint = getattr(x, "_tfrs_amax", None)
  x_amax = None
  if (hint is not None and hint[1] == x._version and hint[2] == x.data_ptr() and x.is_cuda and x.dtype == torch.float32 and
      x.is_contiguous() and x.shape == x0.shape):
    x_amax = hint[0]
  out, out_amax = _Cross.apply(x0, x, W, bias, float(diag_scale), x_amax)
  B, D = out.shape
  if B >= CROSS_TC_MIN_B and D >= CROSS_TC_MIN_D:
    out._tfrs_amax = (out_amax, out._version, out.data_ptr())
  return out


def gemm_tc(a: torch.Tensor, b: torch.Tensor, trans_a: bool = False, trans_b: bool = False) -> torch.Tensor:
  """op(a) @ op(b) on the tensor cores with fp32 parity (split fp16, ~2^-21 relative error); any shape."""
  a = f32c(a, "a"); b = f32c(b, "b")
  M, K = (a.shape[1], a.shape[0]) if trans_a else (a.shape[0], a.shape[1])
  N = b.shape[0] if trans_b else b.shape[1]
  if (b.shape[1] if trans_b else b.shape[0]) != K:
    raise ValueError(f"gemm_tc: inner dimensions differ ({tuple(a.shape)} x {tuple(b.shape)})")
  out = torch.empty((M, N), dtype=torch.float32, device=a.device)
  ws = workspace(lib().tfrs_gemm_tc_workspace_bytes(M, N, K), a.device, "gemm_tc")
  check(lib().tfrs_gemm_tc_f32(int(trans_a), int(trans_b), M, N, K, ptr(a), a.stride(0), ptr(b), b.stride(0), ptr(out), N, ptr(ws),
                               ws.numel(), stream()), "gemm_tc")
  return out


class _CrossLowRank(torch.autograd.Function):
  """x0 * ((x @ U) @ V + bias + diag * x) + x on the tensor cores (forward: 2 GEMMs, formula fused; backward: 4 GEMMs)."""

  @staticmethod
  def forward(ctx, x0, x, U, V, bias, diag_scale):
    x0 = f32c(x0, "x0"); x = f32c(x, "x"); U = f32c(U, "kernel_u"); V = f32c(V, "kernel_v")
    b = None if bias is None else f32c(bias, "bias")
    B, D = x0.shape; p = U.shape[1]
    if U.shape != (D, p) or V.shape != (p, D):
      raise ValueError(f"cross_lowrank: kernels must be [{D},p] and [p,{D}], got {tuple(U.shape)} and {tuple(V.shape)}")
    out = torch.empty_like(x0)
    need_grad = any(ctx.needs_input_grad[:5])
    prod = torch.empty_like(x0) if need_grad else None
    t = torch.empty((B, p), dtype=torch.float32, device=x0.device)
    ws = workspace(lib().tfrs_cross_lowrank_tc_workspace_bytes(B, D, p), x0.device, "cross_lowrank")
    check(lib().tfrs_cross_lowrank_tc_fwd_f32(ptr(x0), ptr(x), ptr(U), ptr(V), ptr(b), B, D, p, D, c_f(diag_scale), ptr(out), ptr(prod),
                                              ptr(t), ptr(ws), ws.numel(), stream()), "cross_lowrank_tc_fwd")
    if need_grad:
      ctx.save_for_backward(x0, x, U, V, t, prod)
    ctx.diag = diag_scale
    ctx.has_bias = b is not None
    return out

  @staticmethod
  def backward(ctx, g):
    x0, x, U, V, t, prod = ctx.saved_tensors
    g = f32c(g, "grad")
    B, D = x0.shape; p = U.shape[1]
    n0, n1, n2, n3, n4 = ctx.needs_input_grad[:5]
    dx0 = torch.empty_like(x0) if n0 else None
    dx = torch.empty_like(x) if n1 else None
    dU = torch.empty_like(U) if n2 else None
    dV = torch.empty_like(V) if n3 else None
    db = torch.empty((D,), dtype=torch.float32, device=x0.device) if (n4 and ctx.has_bias) else None
    ws = workspace(lib().tfrs_cross_lowrank_tc_bwd_workspace_bytes(B, D, p), x0.device, "cross_lowrank_bwd")
    check(lib().tfrs_cross_lowrank_tc_bwd_f32(ptr(x0), ptr(x), ptr(U), ptr(V), ptr(t), ptr(prod), ptr(g), B, D, p, D, c_f(ctx.diag),
                                              ptr(dx0), ptr(dx), ptr(dU), ptr(dV), ptr(db), ptr(ws), ws.numel(), stream()),
          "cross_lowrank_tc_bwd")
    return dx0, dx, dU, dV, db, None


def cross_lowrank_supported(B: int, D: int, p: int) -> bool:
  return B >= CROSS_TC_MIN_B and D >= CROSS_TC_MIN_D and D <= 1024 and 1 <= p <= 1024


def cross_lowrank(x0: torch.Tensor, x: torch.Tensor, U: torch.Tensor, V: torch.Tensor, bias: Optional[torch.Tensor],
                  diag_scale: float = 0.0) -> torch.Tensor:
  """x0 * ((x @ U) @ V + bias + diag_scale * x) + x  (dcn.py:131-148,178-186; multi_layer_dcn.py:146-148)."""
  return _CrossLowRank.apply(x0, x, U, V, bias, float(diag_scale))


# ------------------------------------------------------------------------------------------------
# DotInteraction (DLRM pairwise feature dots)
# ------------------------------------------------------------------------------------------------
class _DotInteraction(torch.autograd.Function):

  @staticmethod
  def forward(ctx, feats, self_interaction, skip_gather):
    feats = f32c(feats, "features")
    B, F, d = feats.shape
    od = lib().tfrs_dot_interaction_out_dim(F, int(self_interaction), int(skip_gather))
    out = torch.empty((B, od), dtype=torch.float32, device=feats.device)
    check(lib().tfrs_dot_interaction_fwd_f32(ptr(feats), B, F, d, int(self_interaction), int(skip_gather), ptr(out), stream()),
          "dot_interaction_fwd")
    ctx.save_for_backward(feats)
    ctx.cfg = (int(self_interaction), int(skip_gather))
    return out

  @staticmethod
  def backward(ctx, g):
    (feats,) = ctx.saved_tensors
    g = f32c(g, "grad")
    B, F, d = feats.shape
    df = torch.empty_like(feats)
    check(lib().tfrs_dot_interaction_bwd_f32(ptr(feats), ptr(g), B, F, d, ctx.cfg[0], ctx.cfg[1], ptr(df), stream()),
          "dot_interaction_bwd")
    return df, None, None


def dot_interaction(feats: torch.Tensor, self_interaction: bool = False, skip_gather: bool = False) -> torch.Tensor:
  """feats [B, F, d] -> pairwise dots, lower triangle (dot_interaction.py:72-104)."""
  return _DotInteraction.apply(feats, bool(self_interaction), bool(skip_gather))


# ------------------------------------------------------------------------------------------------
# K6 Dense layer
# ------------------------------------------------------------------------------------------------
ACT_LINEAR, ACT_RELU, ACT_SIGMOID = 0, 1, 2
DENSE_ACTIVATIONS = {None: ACT_LINEAR, "linear": ACT_LINEAR, "relu": ACT_RELU, "sigmoid": ACT_SIGMOID}


class _Dense(torch.autograd.Function):
  """act(x @ W + bias) with W [in, out]; returns (y, logits) where logits = x @ W + bias for a sigmoid layer (an empty,
  non-differentiable tensor otherwise).  The backward works from the saved OUTPUT y and adds the logits' gradient."""

  @staticmethod
  def forward(ctx, x, W, bias, act):
    x = f32c(x, "x"); W = f32c(W, "kernel")
    b = None if bias is None else f32c(bias, "bias")
    B, K = x.shape
    if W.dim() != 2 or W.shape[0] != K:
      raise ValueError(f"dense: kernel must be [{K}, units], got {tuple(W.shape)}")
    N = W.shape[1]
    if b is not None and b.numel() != N:
      raise ValueError(f"dense: bias must have {N} entries, got {b.numel()}")
    y = torch.empty((B, N), dtype=torch.float32, device=x.device)
    logits = torch.empty((B, N) if act == ACT_SIGMOID else (0,), dtype=torch.float32, device=x.device)
    if B:
      ws = workspace(max(lib().tfrs_dense_fwd_workspace_bytes(B, K, N), 256), x.device, "dense")
      check(lib().tfrs_dense_fwd_f32(ptr(x), ptr(W), ptr(b), B, K, N, act, ptr(y), ptr(logits) if act == ACT_SIGMOID else None,
                                     ptr(ws), ws.numel(), stream()), "dense_fwd")
    ctx.save_for_backward(x, W, y)
    ctx.act = act
    ctx.has_bias = b is not None
    ctx.set_materialize_grads(False)
    if act != ACT_SIGMOID:
      ctx.mark_non_differentiable(logits)
    return y, logits

  @staticmethod
  def backward(ctx, gy, gz):
    x, W, y = ctx.saved_tensors
    B, K = x.shape; N = W.shape[1]
    n0, n1, n2 = ctx.needs_input_grad[:3]
    dx = torch.empty_like(x) if n0 else None
    dW = torch.empty_like(W) if n1 else None
    db = torch.empty((N,), dtype=torch.float32, device=x.device) if (n2 and ctx.has_bias) else None
    if gz is not None and gz.numel() == 0:
      gz = None
    if gy is None and gz is None:
      return None, None, None, None
    if B == 0:
      for t in (dx, dW, db):
        if t is not None:
          t.zero_()
      return dx, dW, db, None
    gy = None if gy is None else f32c(gy, "grad")
    gz = None if gz is None else f32c(gz, "grad_logits")
    ws = workspace(lib().tfrs_dense_bwd_workspace_bytes(B, K, N), x.device, "dense_bwd")
    check(lib().tfrs_dense_bwd_f32(ptr(x), ptr(W), ptr(y), ptr(gy), ptr(gz), B, K, N, ctx.act, ptr(dx), ptr(dW), ptr(db), ptr(ws),
                                   ws.numel(), stream()), "dense_bwd")
    return dx, dW, db, None


def dense_uses_tc(B: int, K: int, N: int) -> bool:
  return bool(lib().tfrs_dense_uses_tc(B, K, N))


def _attach(y: torch.Tensor, attr: str, value: torch.Tensor) -> None:
  """Hangs `value` on `y` as `attr`, valid while `y` is that very tensor, unmodified (its `_version` and `data_ptr`)."""
  setattr(y, attr, (value, y._version, y.data_ptr()))


def _attached(x: torch.Tensor, attr: str, shape) -> Optional[torch.Tensor]:
  """The value `_attach` hung on `x` as `attr`, if it is still valid and has `shape`."""
  hint = getattr(x, attr, None)
  if hint is not None and hint[1] == x._version and hint[2] == x.data_ptr() and tuple(hint[0].shape) == tuple(shape):
    return hint[0]
  return None


def dense(x: torch.Tensor, W: torch.Tensor, bias: Optional[torch.Tensor] = None, activation: Optional[str] = None) -> torch.Tensor:
  """act(x @ W + bias), W [in, out] (tf.keras.layers.Dense); activation None / "linear" / "relu" / "sigmoid" run fused.

  A sigmoid output carries its logits (`_tfrs_logits`, honoured only for that very tensor, unmodified: `_version` +
  `data_ptr` check): the binary cross-entropy of this package then uses the logits form, as tf-keras does with
  `_keras_logits`, and its gradient reaches the logits without passing through the sigmoid."""
  if activation not in DENSE_ACTIVATIONS:
    raise ValueError(f"dense: activation {activation!r} is not fused (use None and apply it afterwards)")
  act = DENSE_ACTIVATIONS[activation]
  lead = x.shape[:-1]
  x2 = x if x.dim() == 2 else x.reshape(-1, x.shape[-1])
  y, z = _Dense.apply(x2, W, bias, act)
  if x.dim() != 2:
    y = y.reshape(*lead, y.shape[-1])
    z = z.reshape(*lead, z.shape[-1]) if act == ACT_SIGMOID else z
  if act == ACT_SIGMOID:
    _attach(y, "_tfrs_logits", z)
  return y


def attached_logits(pred: torch.Tensor) -> Optional[torch.Tensor]:
  """The logits a fused sigmoid Dense attached to `pred`, if `pred` is that very tensor, unmodified."""
  return _attached(pred, "_tfrs_logits", pred.shape)


# ------------------------------------------------------------------------------------------------
# ranking loss + metrics
# ------------------------------------------------------------------------------------------------
LOSS_BCE, LOSS_BCE_LOGITS, LOSS_MSE = 0, 1, 2
REDUCTION_NONE, REDUCTION_SUM, REDUCTION_SUM_OVER_BATCH_SIZE = 0, 1, 2
RANKING_STATS = 5   # [sum w, sum w correct, sum w pred, sum w label, sum w (pred - label)^2], then the AUC buckets


def _flat_weights(sample_weight, B: int, device) -> Optional[torch.Tensor]:
  if sample_weight is None:
    return None
  w = sample_weight if isinstance(sample_weight, torch.Tensor) else torch.as_tensor(sample_weight, dtype=torch.float32)
  w = w.to(device=device, dtype=torch.float32).reshape(-1)
  if w.numel() == 1 and B != 1:
    w = w.expand(B)
  if w.numel() != B:
    raise ValueError(f"sample_weight must have one entry per example (got {w.numel()}, expected {B})")
  return w.contiguous()


class _RankingLoss(torch.autograd.Function):

  @staticmethod
  def forward(ctx, loss_in, labels, weights, kind, reduction, pred, stats, threshold, num_thresholds):
    x = f32c(loss_in, "predictions").reshape(-1)
    B = x.numel()
    y = f32c(labels, "labels").reshape(-1)
    if y.numel() != B:
      raise ValueError(f"labels and predictions must have the same number of entries ({y.numel()} vs {B})")
    w = _flat_weights(weights, B, x.device)
    per = torch.empty((B,), dtype=torch.float32, device=x.device) if reduction == REDUCTION_NONE else None
    loss = torch.empty((1,), dtype=torch.float32, device=x.device) if reduction != REDUCTION_NONE else None
    p = None if pred is None else f32c(pred, "predictions").reshape(-1)
    T = int(num_thresholds) if stats is not None else 0
    ws = workspace(lib().tfrs_ranking_workspace_bytes(B, T), x.device, "ranking")
    check(lib().tfrs_ranking_loss_fwd_f32(ptr(x), ptr(p), ptr(y), ptr(w), B, kind, reduction, ptr(per), ptr(loss), ptr(stats),
                                          c_f(threshold), T, ptr(ws), ws.numel(), stream()), "ranking_loss_fwd")
    ctx.save_for_backward(x, y, w if w is not None else torch.empty(0, device=x.device))
    ctx.has_w = w is not None
    ctx.kind, ctx.reduction, ctx.shape = kind, reduction, loss_in.shape
    return per if reduction == REDUCTION_NONE else loss.view(())

  @staticmethod
  def backward(ctx, g):
    x, y, w = ctx.saved_tensors
    B = x.numel()
    g = f32c(g, "grad").reshape(-1)
    dx = torch.empty_like(x)
    check(lib().tfrs_ranking_loss_bwd_f32(ptr(x), ptr(y), ptr(w) if ctx.has_w else None, B, ctx.kind, ctx.reduction, ptr(g), ptr(dx),
                                          stream()), "ranking_loss_bwd")
    return dx.view(ctx.shape), None, None, None, None, None, None, None, None


def ranking_loss(loss_in: torch.Tensor, labels: torch.Tensor, sample_weight=None, kind: int = LOSS_BCE,
                 reduction: int = REDUCTION_SUM_OVER_BATCH_SIZE, pred: Optional[torch.Tensor] = None,
                 stats: Optional[torch.Tensor] = None, threshold: float = 0.5, num_thresholds: int = 200) -> torch.Tensor:
  """Keras BinaryCrossentropy / MeanSquaredError on [B] or [B, 1] predictions (one example per row): the reduced loss
  (0-dim) or, for REDUCTION_NONE, the weighted per-example losses [B].  `stats` (float64 [RANKING_STATS + 2 T], nullable)
  receives the metric statistics of `pred` from the same launch."""
  return _RankingLoss.apply(loss_in, labels, sample_weight, int(kind), int(reduction), pred, stats, float(threshold),
                            int(num_thresholds))


def ranking_stats_buffer(num_thresholds: int, device) -> torch.Tensor:
  return torch.empty((RANKING_STATS + 2 * int(num_thresholds),), dtype=torch.float64, device=device)


def ranking_metrics(pred: torch.Tensor, labels: torch.Tensor, sample_weight=None, threshold: float = 0.5,
                    num_thresholds: int = 200) -> torch.Tensor:
  """The metric statistics of one batch (layout: include/tfrs_b200.h, ranking loss + metrics) as a float64 device tensor."""
  p = f32c(pred, "predictions").reshape(-1)
  B = p.numel()
  y = f32c(labels, "labels").reshape(-1)
  if y.numel() != B:
    raise ValueError(f"labels and predictions must have the same number of entries ({y.numel()} vs {B})")
  w = _flat_weights(sample_weight, B, p.device)
  stats = ranking_stats_buffer(num_thresholds, p.device)
  ws = workspace(lib().tfrs_ranking_workspace_bytes(B, num_thresholds), p.device, "ranking")
  check(lib().tfrs_ranking_metrics_f32(ptr(p), ptr(y), ptr(w), B, ptr(stats), c_f(threshold), int(num_thresholds), ptr(ws), ws.numel(),
                                       stream()), "ranking_metrics")
  return stats


# ------------------------------------------------------------------------------------------------
# listwise losses + NDCG (K13, csrc/listwise.cu)
# ------------------------------------------------------------------------------------------------
LIST_LOSS_NONE, LIST_LOSS_LISTMLE, LIST_LOSS_PAIRWISE_HINGE, LIST_LOSS_SOFTMAX = 0, 1, 2, 3
LISTWISE_MAX_LIST = 1024
_discounts = {}


def ndcg_discounts(device) -> torch.Tensor:
  """discount[r - 1] = 1 / log2(r + 1) for r = 1 .. LISTWISE_MAX_LIST: computed in float64 on the host, rounded once to fp32."""
  dev = torch.device(device)
  key = dev.index if dev.index is not None else torch.cuda.current_device()
  t = _discounts.get(key)
  if t is None:
    r = np.arange(1, LISTWISE_MAX_LIST + 1, dtype=np.float64)
    t = torch.from_numpy((1.0 / np.log2(r + 1.0)).astype(np.float32)).to(dev)
    _discounts[key] = t
  return t


def _list_tensor(t, name: str, device=None) -> torch.Tensor:
  if not isinstance(t, torch.Tensor):
    t = torch.as_tensor(np.asarray(t), dtype=torch.float32, device=device)
  t = f32c(t, name)
  if t.dim() == 3 and t.shape[-1] == 1:
    t = t.squeeze(-1)
  if t.dim() != 2:
    raise ValueError(f"{name} must be [B, L] or [B, L, 1], got {tuple(t.shape)}")
  return t.contiguous()


def listwise_inputs(predictions, labels, sample_weight=None):
  """(predictions [B, L], labels [B, L], per-list weights [B] or None) as contiguous fp32 device tensors."""
  p = _list_tensor(predictions, "predictions")
  y = _list_tensor(labels, "labels", p.device)
  if y.shape != p.shape:
    raise ValueError(f"labels and predictions must have the same shape ({tuple(y.shape)} vs {tuple(p.shape)})")
  B, L = p.shape
  if not 1 <= L <= LISTWISE_MAX_LIST:
    raise ValueError(f"list length {L} is outside [1, {LISTWISE_MAX_LIST}]")
  w = None
  if sample_weight is not None:
    w = sample_weight if isinstance(sample_weight, torch.Tensor) else torch.as_tensor(np.asarray(sample_weight), dtype=torch.float32)
    w = w.to(device=p.device, dtype=torch.float32)
    if w.dim() == 2 and w.shape[1] > 1:
      raise NotImplementedError("listwise losses and NDCG take one weight per list ([B] or [B, 1]), not per-item weights")
    if w.dim() > 2 or (w.numel() != B and w.numel() != 1):
      raise ValueError(f"sample_weight must be [B] or [B, 1] (got {tuple(w.shape)}, B = {B})")
    w = w.reshape(-1).expand(B).contiguous()
  return p, y, w


def _listwise_fwd(p, y, w, mode, reduction, inv_t, seed, call, dlds, ndcg_stats, topn, ndcg=None):
  B, L = p.shape
  per = torch.empty((B,), dtype=torch.float32, device=p.device) if mode != LIST_LOSS_NONE and reduction == REDUCTION_NONE else None
  loss = torch.empty((1,), dtype=torch.float32, device=p.device) if mode != LIST_LOSS_NONE and reduction != REDUCTION_NONE else None
  disc = ndcg_discounts(p.device) if (ndcg_stats is not None or ndcg is not None) else None
  ws = workspace(lib().tfrs_listwise_workspace_bytes(B, L), p.device, "listwise")
  check(lib().tfrs_listwise_fwd_f32(ptr(p), ptr(y), ptr(w), B, L, mode, reduction, c_f(inv_t), seed & 0xFFFFFFFF, call & 0xFFFFFFFF,
                                    ptr(per), ptr(loss), ptr(dlds), ptr(disc), int(topn or 0), ptr(ndcg), ptr(ndcg_stats), ptr(ws),
                                    ws.numel(), stream()), "listwise_fwd")
  if mode == LIST_LOSS_NONE:
    return None
  return per if reduction == REDUCTION_NONE else loss.view(())


class _ListwiseLoss(torch.autograd.Function):

  @staticmethod
  def forward(ctx, pred, p, y, w, mode, reduction, inv_t, seed, call, ndcg_stats, topn):
    dlds = torch.empty_like(p) if ctx.needs_input_grad[0] else None
    out = _listwise_fwd(p, y, w, mode, reduction, inv_t, seed, call, dlds, ndcg_stats, topn)
    if dlds is not None:
      ctx.save_for_backward(dlds)
    ctx.reduction, ctx.inv_t, ctx.shape = reduction, inv_t, pred.shape
    return out

  @staticmethod
  def backward(ctx, g):
    dlds, = ctx.saved_tensors
    B, L = dlds.shape
    g = f32c(g, "grad").reshape(-1)
    dx = torch.empty_like(dlds)
    check(lib().tfrs_listwise_bwd_f32(ptr(dlds), B, L, ctx.reduction, c_f(ctx.inv_t), ptr(g), ptr(dx), stream()), "listwise_bwd")
    return (dx.view(ctx.shape),) + (None,) * 10


def listwise_loss(predictions: torch.Tensor, labels, sample_weight=None, mode: int = LIST_LOSS_SOFTMAX,
                  reduction: int = REDUCTION_SUM_OVER_BATCH_SIZE, temperature: float = 1.0, seed: int = 0, call: int = 0,
                  ndcg_stats: Optional[torch.Tensor] = None, topn: Optional[int] = None) -> torch.Tensor:
  """A TF-Ranking listwise loss (K13) of [B, L] (or [B, L, 1]) predictions: the reduced loss (0-dim) or, for REDUCTION_NONE,
  the weighted per-list losses [B].  `ndcg_stats` (float64 [2], nullable) receives [sum w ndcg, sum w] at `topn` from the same
  launch.  Differentiable in `predictions`; the backward is one scaling launch."""
  if mode == LIST_LOSS_NONE:
    raise ValueError("listwise_loss needs a loss mode")
  if not temperature > 0 or not np.isfinite(temperature):
    raise ValueError(f"temperature must be finite and > 0, got {temperature}")
  p, y, w = listwise_inputs(predictions, labels, sample_weight)
  inv_t = float(np.float32(1.0 / float(temperature)))
  return _ListwiseLoss.apply(predictions, p, y, w, int(mode), int(reduction), inv_t, int(seed), int(call), ndcg_stats, topn)


def ndcg_stats_buffer(device) -> torch.Tensor:
  return torch.empty((2,), dtype=torch.float64, device=device)


@torch.no_grad()
def listwise_ndcg(predictions: torch.Tensor, labels, sample_weight=None, topn: Optional[int] = None, per_list: bool = False):
  """The NDCG statistics [sum w ndcg, sum w] of one batch (float64 device tensor) from K13's metric-only launch; with
  per_list=True also every list's NDCG [B] (fp32)."""
  p, y, w = listwise_inputs(predictions, labels, sample_weight)
  stats = ndcg_stats_buffer(p.device)
  nd = torch.empty((p.shape[0],), dtype=torch.float32, device=p.device) if per_list else None
  _listwise_fwd(p, y, w, LIST_LOSS_NONE, REDUCTION_SUM, 1.0, 0, 0, None, stats, topn, nd)
  return (stats, nd) if per_list else stats


# ------------------------------------------------------------------------------------------------
# K15 vocabulary lookup: the hash tables of layers.StringLookup / IntegerLookup
# ------------------------------------------------------------------------------------------------
class _LookupTableDesc(ctypes.Structure):
  _fields_ = [("keys", ctypes.c_void_p), ("offsets", ctypes.c_void_p), ("V", ctypes.c_int64), ("kind", ctypes.c_int32),
              ("has_mask", ctypes.c_int32), ("mask", ctypes.c_int64), ("mask_bytes", ctypes.c_void_p),
              ("mask_len", ctypes.c_int64), ("slots", ctypes.c_void_p)]


class LookupTable(NamedTuple):
  """A built vocabulary table: int64 `keys` [V], or uint8 string bytes with int64 `offsets` [V+1]; `mask` is the int mask
  token or the uint8 bytes of the string one (None: no mask); `slots` is the table memory the build filled."""
  keys: torch.Tensor
  offsets: Optional[torch.Tensor]
  mask: object
  slots: torch.Tensor

  @property
  def size(self) -> int:
    return self.keys.numel() if self.offsets is None else self.offsets.numel() - 1

  def desc(self) -> _LookupTableDesc:
    d = _LookupTableDesc()
    d.keys, d.V, d.slots = self.keys.data_ptr(), self.size, self.slots.data_ptr()
    d.kind = _ffi.I64 if self.offsets is None else _ffi.BYTES
    if self.offsets is not None:
      d.offsets = self.offsets.data_ptr()
    if self.mask is not None:
      d.has_mask = 1
      if self.offsets is None:
        d.mask = int(self.mask)
      else:
        d.mask_bytes, d.mask_len = self.mask.data_ptr(), self.mask.numel()
    return d


def lookup_build(keys: torch.Tensor, offsets: Optional[torch.Tensor] = None, mask=None) -> LookupTable:
  """Builds the table of a vocabulary on its device: CUDA int64 `keys` [V], or the uint8 bytes of V strings with their int64
  `offsets` [V+1].  `mask` is the mask token (an int, or a CUDA uint8 tensor of the string's bytes) or None.  Raises
  ValueError when two keys are equal; that check is the only host read (4 bytes) of the build."""
  require_cuda(keys, "keys")
  if offsets is None:
    if keys.dtype != torch.int64 or keys.dim() != 1:
      raise TypeError("lookup_build: integer keys must be a 1-D int64 tensor")
    kind, V = _ffi.I64, keys.numel()
  else:
    require_cuda(offsets, "offsets")
    if keys.dtype != torch.uint8 or offsets.dtype != torch.int64 or offsets.dim() != 1 or offsets.numel() < 1:
      raise TypeError("lookup_build: string keys must be uint8 bytes with 1-D int64 offsets [V+1]")
    if mask is not None:
      require_cuda(mask, "mask")
      if mask.dtype != torch.uint8:
        raise TypeError("lookup_build: the string mask token must be uint8 bytes")
      mask = mask.contiguous()
    kind, V = _ffi.BYTES, offsets.numel() - 1
  nb = lib().tfrs_lookup_table_bytes(V, kind)
  if nb == 0:
    raise ValueError(f"lookup_build: {V} keys; a table holds fewer than 2^30")
  table = LookupTable(keys.contiguous(), None if offsets is None else offsets.contiguous(), mask,
                      torch.empty((nb,), dtype=torch.uint8, device=keys.device))
  dup = torch.empty((1,), dtype=torch.int32, device=keys.device)
  desc = table.desc()
  check(lib().tfrs_lookup_build(ctypes.byref(desc), ptr(dup), stream()), "lookup_build")
  if int(dup.item()):
    raise ValueError("lookup_build: the vocabulary has duplicate entries")
  return table


def lookup(table: LookupTable, values, base: int, oov: Optional[int]) -> torch.Tensor:
  """int64 index of every value, in the values' shape: 0 for the mask token, base + p for vocabulary key p, `oov` for any
  other value.  `values` is a CUDA int32 / int64 tensor (integer tables) or a (uint8 bytes, int64 offsets [n+1]) pair of
  CUDA tensors (string tables, 1-D output).  With oov=None a value outside the vocabulary raises ValueError, which costs
  one 4-byte read; otherwise the call never reads device memory on the host.  One launch."""
  values, offsets = values if isinstance(values, tuple) else (values, None)
  kind = _value_kind(values, offsets)
  values = values.contiguous()
  offsets = offsets.contiguous() if offsets is not None else None
  n = values.numel() if offsets is None else offsets.numel() - 1
  out = torch.empty(values.shape if offsets is None else (n,), dtype=torch.int64, device=values.device)
  if n == 0:
    return out
  miss = torch.zeros((1,), dtype=torch.int32, device=values.device) if oov is None else None
  desc = table.desc()
  check(lib().tfrs_lookup(ctypes.byref(desc), ptr(values), ptr(offsets), kind, n, int(base), -1 if oov is None else int(oov),
                          ptr(miss), ptr(out), stream()), "lookup")
  if miss is not None and int(miss.item()):
    raise ValueError("lookup: a value is not in the vocabulary, and there is no out-of-vocabulary index "
                     "(num_oov_indices=0)")
  return out


def lookup_invert(idx: torch.Tensor, size: int, base: int, keys: Optional[torch.Tensor], mask_out: Optional[int],
                  oov_out: int) -> torch.Tensor:
  """int64 [idx's shape]: keys[x - base] for an index x in [base, base + size) (x - base when keys is None), mask_out for
  x == 0 when mask_out is not None, oov_out for every other x.  One launch."""
  require_cuda(idx, "indices")
  kind = _ffi.ids_dtype_code(idx)
  idx = idx.contiguous()
  out = torch.empty(idx.shape, dtype=torch.int64, device=idx.device)
  if keys is not None:
    require_cuda(keys, "keys")
    if keys.dtype != torch.int64 or keys.numel() != size:
      raise ValueError("lookup_invert: keys must be int64 [size]")
  check(lib().tfrs_lookup_invert(ptr(idx), kind, idx.numel(), ptr(keys), int(size), int(base), int(mask_out is not None),
                                 0 if mask_out is None else int(mask_out), int(oov_out), ptr(out), stream()),
        "lookup_invert")
  return out


def launch_count() -> int:
  return int(lib().tfrs_launch_count())


# ------------------------------------------------------------------------------------------------
# K16 text vectorization: layers.TextVectorization on the K15 table of its inner StringLookup
# ------------------------------------------------------------------------------------------------
TEXT_LOWER, TEXT_STRIP = 1, 2


def _text_standardize(data: torch.Tensor, offsets: torch.Tensor, flags: int, with_max: bool):
  n = offsets.numel() - 1
  scratch = torch.empty_like(data)
  counts = torch.empty((n,), dtype=torch.int32, device=offsets.device)
  mx = torch.empty((1,), dtype=torch.int32, device=offsets.device) if with_max else None
  check(lib().tfrs_text_standardize(ptr(data), ptr(offsets), n, data.numel(), int(flags), ptr(scratch), ptr(counts),
                                    ptr(mx), stream()), "text_standardize")
  return scratch, counts, mx


def text_vectorize(table: LookupTable, data: torch.Tensor, offsets: torch.Tensor, flags: int, T: Optional[int], base: int,
                   oov: int) -> torch.Tensor:
  """int64 [n, T]: the tokens of n strings (uint8 `data`, int64 `offsets` [n+1] on the device), standardized by `flags`
  (TEXT_LOWER | TEXT_STRIP) and split on ASCII whitespace, each looked up in the string table: base + p for vocabulary
  entry p, `oov` for any other token, 0 after a string's last token.  T=None takes the longest token count, at the cost
  of one 4-byte host read; with T given, the call never reads device memory on the host.  Two launches."""
  if table.offsets is None:
    raise TypeError("text_vectorize: the table must be a string table")
  scratch, _, mx = _text_standardize(data, offsets, flags, T is None)
  if T is None:
    T = int(mx.item())
  out = torch.empty((offsets.numel() - 1, T), dtype=torch.int64, device=offsets.device)
  desc = table.desc()
  check(lib().tfrs_text_lookup(ctypes.byref(desc), ptr(scratch), ptr(offsets), out.shape[0], T, int(base), int(oov),
                               ptr(out), stream()), "text_lookup")
  return out


def text_tokens(data: torch.Tensor, offsets: torch.Tensor, flags: int) -> Tuple[np.ndarray, np.ndarray]:
  """The tokens of n strings as text_vectorize finds them, for adapt: (standardized bytes, int64 [tokens, 2] of (offset,
  length) into them, string by string), both read back to the host."""
  scratch, counts, _ = _text_standardize(data, offsets, flags, False)
  tok_off = np.zeros(counts.numel() + 1, np.int64)
  np.cumsum(counts.cpu().numpy(), out=tok_off[1:])
  spans = torch.empty((int(tok_off[-1]), 2), dtype=torch.int64, device=offsets.device)
  tok_off_d = torch.from_numpy(tok_off).to(offsets.device)
  check(lib().tfrs_text_spans(ptr(scratch), ptr(offsets), counts.numel(), ptr(tok_off_d), ptr(spans), stream()),
        "text_spans")
  return scratch.cpu().numpy(), spans.cpu().numpy()


# ------------------------------------------------------------------------------------------------
# K17 numeric columns and pooling: layers.Discretization, layers.Normalization, layers.GlobalAveragePooling1D
# ------------------------------------------------------------------------------------------------
_VALUE_KINDS = {torch.int32: _ffi.I32, torch.int64: _ffi.I64, torch.float32: _ffi.F32, torch.float64: _ffi.F64}
_MASK_KINDS = {torch.int32: _ffi.I32, torch.int64: _ffi.I64, torch.bool: _ffi.BOOL}


def _numeric(x: torch.Tensor, what: str) -> Tuple[torch.Tensor, int]:
  require_cuda(x, what)
  if x.dtype not in _VALUE_KINDS:
    raise TypeError(f"{what}: values must be int32, int64, float32 or float64, got {x.dtype}")
  return x.contiguous(), _VALUE_KINDS[x.dtype]


def bucketize(x: torch.Tensor, boundaries: torch.Tensor) -> torch.Tensor:
  """int64 [x's shape]: the number of float32 `boundaries` (sorted, CUDA) at or below each value; NaN gives their count.
  Integers are rounded to float32 first; float64 values are compared as doubles.  One launch."""
  x, kind = _numeric(x, "bucketize")
  require_cuda(boundaries, "boundaries")
  if boundaries.dtype != torch.float32 or boundaries.dim() != 1:
    raise TypeError("bucketize: boundaries must be a 1-D float32 tensor")
  b = boundaries.contiguous()
  out = torch.empty(x.shape, dtype=torch.int64, device=x.device)
  check(lib().tfrs_bucketize(ptr(x), kind, x.numel(), ptr(b), b.numel(), ptr(out), stream()), "bucketize")
  return out


def normalize(x: torch.Tensor, mean: torch.Tensor, var: torch.Tensor, invert: bool = False) -> torch.Tensor:
  """float32 [x's shape]: (f32(x) - mean) / max(sqrt(var), 1e-7), or mean + f32(x) * max(sqrt(var), 1e-7) with invert;
  `mean` and `var` are float32 [C] (CUDA), C = 1 or x's last dimension.  One launch."""
  x, kind = _numeric(x, "normalize")
  C = mean.numel()
  if mean.dtype != torch.float32 or var.dtype != torch.float32 or var.numel() != C or C < 1:
    raise TypeError("normalize: mean and variance must be float32 tensors of one size C >= 1")
  if C > 1 and (x.dim() == 0 or x.shape[-1] != C):
    raise ValueError(f"normalize: {C} statistics for an input of shape {tuple(x.shape)}")
  out = torch.empty(x.shape, dtype=torch.float32, device=x.device)
  check(lib().tfrs_normalize(ptr(x), kind, x.numel(), C, ptr(mean.contiguous()), ptr(var.contiguous()), int(bool(invert)),
                             ptr(out), stream()), "normalize")
  return out


def normalization_adapt(x: torch.Tensor, C: int, batch_rows: int, state: torch.Tensor, count: torch.Tensor) -> None:
  """Merges the batches of `batch_rows` rows of x (axis 0; channel = last index mod C) into `state` (float32 [2, C]: mean,
  variance) and `count` (int64 [1]) in place, as Keras's Normalization.adapt does.  One launch for a single batch, two
  otherwise; nothing is read on the host."""
  x, kind = _numeric(x, "normalization_adapt")
  if state.dtype != torch.float32 or state.shape != (2, C) or count.dtype != torch.int64 or count.numel() != 1:
    raise TypeError("normalization_adapt: state must be float32 [2, C] and count int64 [1]")
  N = x.shape[0] if x.dim() else 1
  R = x.numel() // N if N else 1
  nb = lib().tfrs_normalization_adapt_workspace_bytes(N, C, batch_rows)
  ws = workspace(nb, x.device, "normalization_adapt") if nb else None
  check(lib().tfrs_normalization_adapt(ptr(x), kind, N, R, C, batch_rows, ptr(state), ptr(count), ptr(ws), nb, stream()),
        "normalization_adapt")


def _mask_arg(mask: Optional[torch.Tensor], shape, op: str, name: str = "the mask"):
  """(mask, kind) for a kernel's (const void* mask, int mask_kind): a Keras mask (bool / int32 / int64, CUDA, nonzero =
  kept) of exactly `shape`, made contiguous; (None, 0) for no mask."""
  if mask is None:
    return None, 0
  require_cuda(mask, name)
  if mask.dtype not in _MASK_KINDS:
    raise TypeError(f"{op}: {name} must be bool, int32 or int64, got {mask.dtype}")
  if tuple(mask.shape) != tuple(shape):
    raise ValueError(f"{op}: {name} has shape {tuple(mask.shape)}, expected {tuple(shape)}")
  return mask.contiguous(), _MASK_KINDS[mask.dtype]


class _MeanPool(torch.autograd.Function):

  @staticmethod
  def forward(ctx, x, mask):
    B, T, d = x.shape
    m, mk = _mask_arg(mask, (B, T), "mean_pool")
    out = torch.empty((B, d), dtype=torch.float32, device=x.device)
    check(lib().tfrs_mean_pool_fwd(ptr(x), B, T, d, x.stride(0), x.stride(1), x.stride(2), ptr(m), mk, ptr(out),
                                   stream()), "mean_pool_fwd")
    ctx.save_for_backward(m)
    ctx.shape, ctx.mk = (B, T, d), mk
    return out

  @staticmethod
  def backward(ctx, g):
    (m,) = ctx.saved_tensors
    B, T, d = ctx.shape
    g = g.to(torch.float32).contiguous()
    dx = torch.empty((B, T, d), dtype=torch.float32, device=g.device)
    check(lib().tfrs_mean_pool_bwd(ptr(g), B, T, d, ptr(m), ctx.mk, ptr(dx), stream()), "mean_pool_bwd")
    return dx, None


def mean_pool(x: torch.Tensor, mask: Optional[torch.Tensor] = None) -> torch.Tensor:
  """float32 [B, d]: the mean over t of x [B, T, d] (float32, any strides), counting only the positions where `mask` ([B,
  T] bool / int32 / int64, CUDA) is nonzero; an all-masked row is 0/0.  Products and sums in float32, t ascending from
  +0.0f.  Backward: dx = f32(g / count) * mask, or g / T.  One launch each way."""
  require_cuda(x, "inputs")
  if x.dtype != torch.float32 or x.dim() != 3:
    raise TypeError(f"mean_pool: inputs must be float32 [B, T, d], got {x.dtype} {tuple(x.shape)}")
  return _MeanPool.apply(x, mask)


def attached_mask(x: torch.Tensor) -> Optional[torch.Tensor]:
  """The mask (the ids, nonzero = kept) an Embedding with mask_zero=True attached to its output `x`, if `x` is that very
  tensor, unmodified."""
  return _attached(x, "_tfrs_mask", x.shape[:-1])


def attach_mask(y: torch.Tensor, mask: Optional[torch.Tensor]) -> torch.Tensor:
  """Attaches `mask` (y.shape[:-1], nonzero = kept) to a layer's output `y` for `attached_mask`; None attaches nothing.
  Returns `y`."""
  if mask is not None:
    _attach(y, "_tfrs_mask", mask)
  return y


def layer_mask(x: torch.Tensor, mask=None) -> Optional[torch.Tensor]:
  """The mask a layer applies to its input `x`: `mask` when one is passed (an array or list becomes a tensor on x's
  device), else the mask attached to `x`, if any."""
  if mask is None:
    return attached_mask(x)
  if isinstance(mask, torch.Tensor):
    return mask
  return torch.from_numpy(np.ascontiguousarray(mask)).to(x.device)


# ------------------------------------------------------------------------------------------------
# K19 GRU recurrence: layers.GRU (reset_after=True); the input projection runs on K6
# ------------------------------------------------------------------------------------------------
GRU_MAX_UNITS = 2048   # TFRS_GRU_MAX_UNITS of include/tfrs_b200.h


def _gru_fwd(gx, U, b_r, h0, m, mk, return_sequences: bool, save: bool):
  B, T, u3 = gx.shape
  u = u3 // 3
  new = lambda *shape: torch.empty(shape, dtype=torch.float32, device=gx.device)
  seq = new(B, T, u) if return_sequences else None
  h_last = new(B, u)
  gates, h_prev = (new(B, T, 4 * u), new(B, T, u)) if save else (None, None)
  check(lib().tfrs_gru_fwd_f32(ptr(gx), ptr(U), ptr(b_r), ptr(h0), ptr(m), mk, B, T, u, ptr(seq), ptr(h_last), ptr(gates),
                               ptr(h_prev), stream()), "gru_fwd")
  return seq, h_last, gates, h_prev


class _GRURecurrence(torch.autograd.Function):
  """(out_seq, h_T) with return_sequences, else h_T alone, from gx = x.W + b_i [B, T, 3u]; differentiable in gx, U, b_r
  and h0."""

  @staticmethod
  def forward(ctx, gx, U, b_r, h0, m, mk, return_sequences):
    seq, h_last, gates, h_prev = _gru_fwd(gx, U, b_r, h0, m, mk, return_sequences, True)
    ctx.save_for_backward(U, gates, h_prev, m)
    ctx.mk, ctx.return_sequences = mk, return_sequences
    ctx.set_materialize_grads(False)
    return (seq, h_last) if return_sequences else h_last

  @staticmethod
  def backward(ctx, *grads):
    U, gates, h_prev, m = ctx.saved_tensors
    g_seq, g_last = grads if ctx.return_sequences else (None, grads[0])
    B, T, u = h_prev.shape
    n_gx, n_U, n_br, n_h0 = ctx.needs_input_grad[:4]
    new = lambda *shape: torch.empty(shape, dtype=torch.float32, device=U.device)
    dgx = new(B, T, 3 * u)
    dU = new(u, 3 * u) if n_U else None
    db_r = new(3 * u) if n_br else None
    dh0 = new(B, u) if n_h0 else None
    if B == 0 or (g_seq is None and g_last is None):
      for t in (dgx, dU, db_r, dh0):
        if t is not None:
          t.zero_()
    else:
      g_seq = None if g_seq is None else f32c(g_seq, "grad")
      g_last = None if g_last is None else f32c(g_last, "grad")
      ws = workspace(lib().tfrs_gru_bwd_workspace_bytes(B, T, u), U.device, "gru_bwd")
      check(lib().tfrs_gru_bwd_f32(ptr(U), ptr(gates), ptr(h_prev), ptr(m), ctx.mk, ptr(g_seq), ptr(g_last), B, T, u,
                                   ptr(dgx), ptr(dU), ptr(db_r), ptr(dh0), ptr(ws), ws.numel(), stream()), "gru_bwd")
    return dgx if n_gx else None, dU, db_r, dh0, None, None, None


def gru(x: torch.Tensor, kernel: torch.Tensor, recurrent_kernel: torch.Tensor, bias: Optional[torch.Tensor] = None,
        initial_state: Optional[torch.Tensor] = None, mask: Optional[torch.Tensor] = None,
        return_sequences: bool = False) -> Tuple[torch.Tensor, torch.Tensor]:
  """tf.keras.layers.GRU(reset_after=True) over x [B, T, D]: returns (output, h_T), output = [B, T, u] every h_t with
  `return_sequences`, else h_T [B, u].  kernel W [D, 3u], recurrent_kernel U [u, 3u] and bias [2, 3u] = (b_i, b_r) as
  Keras stores them, columns (z, r, h); initial_state h_0 [B, u] (zeros when None); mask [B, T] bool / int32 / int64
  (nonzero = kept): a masked step carries h unchanged.  gx = x.W + b_i is one K6 Dense call (ops.dense), the T steps are
  one K19 launch; the backward is K19's reverse launch plus K6's backward for the projection and for dU, db_r.
  Differentiable in x, all three weights and initial_state."""
  require_cuda(x, "inputs")
  if x.dim() != 3:
    raise ValueError(f"gru: inputs must be [batch, timesteps, features], got shape {tuple(x.shape)}")
  B, T, D = x.shape
  if T == 0:
    raise ValueError("gru: the inputs have no time steps (T = 0)")
  require_cuda(recurrent_kernel, "recurrent_kernel")
  u = recurrent_kernel.shape[0] if recurrent_kernel.dim() == 2 else 0
  if recurrent_kernel.dim() != 2 or recurrent_kernel.shape[1] != 3 * u or u == 0:
    raise ValueError(f"gru: recurrent_kernel must be [units, 3 * units], got {tuple(recurrent_kernel.shape)}")
  if u > GRU_MAX_UNITS:
    raise ValueError(f"gru: units = {u} is above the kernel's ceiling of {GRU_MAX_UNITS}")
  if tuple(kernel.shape) != (D, 3 * u):
    raise ValueError(f"gru: kernel must be [{D}, {3 * u}], got {tuple(kernel.shape)}")
  if bias is not None and tuple(bias.shape) != (2, 3 * u):
    raise ValueError(f"gru: bias must be [2, {3 * u}] (reset_after=True), got {tuple(bias.shape)}")
  if initial_state is not None and tuple(initial_state.shape) != (B, u):
    raise ValueError(f"gru: initial_state must be [{B}, {u}], got {tuple(initial_state.shape)}")
  if mask is not None and return_sequences:
    raise NotImplementedError("gru: a mask together with return_sequences=True is not supported")
  m, mk = _mask_arg(mask, (B, T), "gru")
  gx = dense(x.reshape(B * T, D), kernel, None if bias is None else bias[0]).reshape(B, T, 3 * u)
  U = f32c(recurrent_kernel, "recurrent_kernel")
  b_r = None if bias is None else f32c(bias[1], "bias")
  h0 = None if initial_state is None else f32c(initial_state, "initial_state")
  if torch.is_grad_enabled() and any(t is not None and t.requires_grad for t in (gx, U, b_r, h0)):
    out = _GRURecurrence.apply(gx, U, b_r, h0, m, mk, bool(return_sequences))
    return out if return_sequences else (out, out)
  seq, h_last, _, _ = _gru_fwd(gx.detach(), U.detach(), None if b_r is None else b_r.detach(),
                               None if h0 is None else h0.detach(), m, mk, bool(return_sequences), False)
  return (seq if return_sequences else h_last), h_last


# ------------------------------------------------------------------------------------------------
# K20 LSTM recurrence: layers.LSTM; the input projection runs on K6
# ------------------------------------------------------------------------------------------------
LSTM_MAX_UNITS = 2048   # TFRS_LSTM_MAX_UNITS of include/tfrs_b200.h


def _lstm_fwd(gx, U, h0, c0, m, mk, return_sequences: bool, save: bool):
  B, T, u4 = gx.shape
  u = u4 // 4
  new = lambda *shape: torch.empty(shape, dtype=torch.float32, device=gx.device)
  seq = new(B, T, u) if return_sequences else None
  h_last, c_last = new(B, u), new(B, u)
  gates, c_seq, h_prev = (new(B, T, 4 * u), new(B, T, u), new(B, T, u)) if save else (None, None, None)
  check(lib().tfrs_lstm_fwd_f32(ptr(gx), ptr(U), ptr(h0), ptr(c0), ptr(m), mk, B, T, u, ptr(seq), ptr(h_last),
                                ptr(c_last), ptr(gates), ptr(c_seq), ptr(h_prev), stream()), "lstm_fwd")
  return seq, h_last, c_last, gates, c_seq, h_prev


class _LSTMRecurrence(torch.autograd.Function):
  """(out_seq, h_T, c_T) with return_sequences, else (h_T, c_T), from gx = x.W + b [B, T, 4u]; differentiable in gx, U,
  h0 and c0."""

  @staticmethod
  def forward(ctx, gx, U, h0, c0, m, mk, return_sequences):
    seq, h_last, c_last, gates, c_seq, h_prev = _lstm_fwd(gx, U, h0, c0, m, mk, return_sequences, True)
    ctx.save_for_backward(U, gates, c_seq, h_prev, c0, m)
    ctx.mk, ctx.return_sequences = mk, return_sequences
    ctx.set_materialize_grads(False)
    return (seq, h_last, c_last) if return_sequences else (h_last, c_last)

  @staticmethod
  def backward(ctx, *grads):
    U, gates, c_seq, h_prev, c0, m = ctx.saved_tensors
    g_seq, g_h, g_c = grads if ctx.return_sequences else (None, *grads)
    B, T, u = h_prev.shape
    n_gx, n_U, n_h0, n_c0 = ctx.needs_input_grad[:4]
    new = lambda *shape: torch.empty(shape, dtype=torch.float32, device=U.device)
    dz = new(B, T, 4 * u)
    dU = new(u, 4 * u) if n_U else None
    dh0 = new(B, u) if n_h0 else None
    dc0 = new(B, u) if n_c0 else None
    if B == 0 or (g_seq is None and g_h is None and g_c is None):
      for t in (dz, dU, dh0, dc0):
        if t is not None:
          t.zero_()
    else:
      g_seq, g_h, g_c = (None if g is None else f32c(g, "grad") for g in (g_seq, g_h, g_c))
      ws = workspace(lib().tfrs_lstm_bwd_workspace_bytes(B, T, u), U.device, "lstm_bwd")
      check(lib().tfrs_lstm_bwd_f32(ptr(U), ptr(gates), ptr(c_seq), ptr(h_prev), ptr(c0), ptr(m), ctx.mk, ptr(g_seq),
                                    ptr(g_h), ptr(g_c), B, T, u, ptr(dz), ptr(dU), ptr(dh0), ptr(dc0), ptr(ws),
                                    ws.numel(), stream()), "lstm_bwd")
    return dz if n_gx else None, dU, dh0, dc0, None, None, None


def lstm(x: torch.Tensor, kernel: torch.Tensor, recurrent_kernel: torch.Tensor, bias: Optional[torch.Tensor] = None,
         initial_state: Optional[Sequence[torch.Tensor]] = None, mask: Optional[torch.Tensor] = None,
         return_sequences: bool = False) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
  """tf.keras.layers.LSTM over x [B, T, D]: returns (output, h_T, c_T), output = [B, T, u] every h_t with
  `return_sequences`, else h_T [B, u].  kernel W [D, 4u], recurrent_kernel U [u, 4u] and bias [4u] as Keras stores them,
  columns (i, f, c, o); initial_state (h_0, c_0), each [B, u] (zeros when None); mask [B, T] bool / int32 / int64
  (nonzero = kept): a masked step carries h and c unchanged.  gx = x.W + b is one K6 Dense call (ops.dense), the T steps
  are one K20 launch; the backward is K20's reverse launch plus K6's backward for the projection and for dU.
  Differentiable in x, all three weights and both initial states."""
  require_cuda(x, "inputs")
  if x.dim() != 3:
    raise ValueError(f"lstm: inputs must be [batch, timesteps, features], got shape {tuple(x.shape)}")
  B, T, D = x.shape
  if T == 0:
    raise ValueError("lstm: the inputs have no time steps (T = 0)")
  require_cuda(recurrent_kernel, "recurrent_kernel")
  u = recurrent_kernel.shape[0] if recurrent_kernel.dim() == 2 else 0
  if recurrent_kernel.dim() != 2 or recurrent_kernel.shape[1] != 4 * u or u == 0:
    raise ValueError(f"lstm: recurrent_kernel must be [units, 4 * units], got {tuple(recurrent_kernel.shape)}")
  if u > LSTM_MAX_UNITS:
    raise ValueError(f"lstm: units = {u} is above the kernel's ceiling of {LSTM_MAX_UNITS}")
  if tuple(kernel.shape) != (D, 4 * u):
    raise ValueError(f"lstm: kernel must be [{D}, {4 * u}], got {tuple(kernel.shape)}")
  if bias is not None and tuple(bias.shape) != (4 * u,):
    raise ValueError(f"lstm: bias must be [{4 * u}], got {tuple(bias.shape)}")
  h0 = c0 = None
  if initial_state is not None:
    if isinstance(initial_state, torch.Tensor) or len(initial_state) != 2:
      raise ValueError("lstm: initial_state must be the pair (h_0, c_0)")
    for name, s in zip(("h_0", "c_0"), initial_state):
      if tuple(s.shape) != (B, u):
        raise ValueError(f"lstm: initial_state {name} must be [{B}, {u}], got {tuple(s.shape)}")
    h0, c0 = (f32c(s, "initial_state") for s in initial_state)
  if mask is not None and return_sequences:
    raise NotImplementedError("lstm: a mask together with return_sequences=True is not supported")
  m, mk = _mask_arg(mask, (B, T), "lstm")
  gx = dense(x.reshape(B * T, D), kernel, bias).reshape(B, T, 4 * u)
  U = f32c(recurrent_kernel, "recurrent_kernel")
  if torch.is_grad_enabled() and any(t is not None and t.requires_grad for t in (gx, U, h0, c0)):
    out = _LSTMRecurrence.apply(gx, U, h0, c0, m, mk, bool(return_sequences))
    return out if return_sequences else (out[0], out[0], out[1])
  seq, h_last, c_last, _, _, _ = _lstm_fwd(gx.detach(), U.detach(), None if h0 is None else h0.detach(),
                                           None if c0 is None else c0.detach(), m, mk, bool(return_sequences), False)
  return (seq if return_sequences else h_last), h_last, c_last


# ------------------------------------------------------------------------------------------------
# K21 attention core: layers.MultiHeadAttention; the four projections run on K6
# ------------------------------------------------------------------------------------------------
MHA_MAX_HEAD_DIM = 128   # TFRS_MHA_MAX_HEAD_DIM of include/tfrs_b200.h


class _MhaMasks(ctypes.Structure):
  _fields_ = [("query", c_p), ("query_kind", c_i), ("value", c_p), ("value_kind", c_i), ("key", c_p), ("key_kind", c_i),
              ("attention", c_p), ("attention_kind", c_i), ("causal", c_i)]


def _mha_masks(masks, causal: bool) -> _MhaMasks:
  """masks: the query, value, key and attention masks as _mask_arg's (mask, kind) pairs."""
  s = _MhaMasks()
  for name, (m, kind) in zip(("query", "value", "key", "attention"), masks):
    setattr(s, name, ptr(m))
    setattr(s, name + "_kind", kind)
  s.causal = int(bool(causal))
  return s


def _attention_fwd(Q, K, V, H, dk, dv, masks, causal, want_p, save):
  B, T, S = Q.shape[0], Q.shape[1], K.shape[1]
  O = torch.empty((B, T, H * dv), dtype=torch.float32, device=Q.device)
  stats = torch.empty((B, H, T, 2), dtype=torch.float32, device=Q.device) if save else None
  P = torch.empty((B, H, T, S), dtype=torch.float32, device=Q.device) if want_p else None
  m = _mha_masks(masks, causal)
  check(lib().tfrs_mha_fwd_f32(ptr(Q), ptr(K), ptr(V), ctypes.byref(m), B, T, S, H, dk, dv, ptr(O), ptr(stats), ptr(P),
                               stream()), "mha_fwd")
  return O, stats, P


class _AttentionCore(torch.autograd.Function):
  """(O [B, T, H*dv], P [B, H, T, S] or an empty tensor) from the projected Q, K, V; differentiable in Q, K and V.  P is
  not differentiable."""

  @staticmethod
  def forward(ctx, Q, K, V, H, dk, dv, masks, causal, want_p):
    O, stats, P = _attention_fwd(Q, K, V, H, dk, dv, masks, causal, want_p, True)
    P = P if want_p else torch.empty((0,), dtype=torch.float32, device=Q.device)
    ctx.save_for_backward(Q, K, V, O, stats, *(m for m, _ in masks))
    ctx.shape, ctx.causal, ctx.kinds = (H, dk, dv), causal, [kind for _, kind in masks]
    ctx.mark_non_differentiable(P)
    ctx.set_materialize_grads(False)
    return O, P

  @staticmethod
  def backward(ctx, dO, _dP):
    Q, K, V, O, stats, *masks = ctx.saved_tensors
    H, dk, dv = ctx.shape
    B, T, S = Q.shape[0], Q.shape[1], K.shape[1]
    dQ, dK, dV = torch.empty_like(Q), torch.empty_like(K), torch.empty_like(V)
    if dO is None or B == 0:
      for t in (dQ, dK, dV):
        t.zero_()
    else:
      dO = f32c(dO, "grad")
      m = _mha_masks(zip(masks, ctx.kinds), ctx.causal)
      ws = workspace(lib().tfrs_mha_bwd_workspace_bytes(B, T, H), Q.device, "mha_bwd")
      check(lib().tfrs_mha_bwd_f32(ptr(Q), ptr(K), ptr(V), ctypes.byref(m), ptr(O), ptr(stats), ptr(dO), B, T, S, H, dk,
                                   dv, ptr(dQ), ptr(dK), ptr(dV), ptr(ws), ws.numel(), stream()), "mha_bwd")
    n = ctx.needs_input_grad
    return (dQ if n[0] else None, dK if n[1] else None, dV if n[2] else None) + (None,) * 6


def attention_core(Q: torch.Tensor, K: torch.Tensor, V: torch.Tensor, num_heads: int, query_mask=None, value_mask=None,
                   key_mask=None, attention_mask=None, causal: bool = False, return_scores: bool = False):
  """K21 on projected tensors: Q [B, T, H*dk], K [B, S, H*dk], V [B, S, H*dv] (float32, CUDA) -> (O [B, T, H*dv],
  P [B, H, T, S] with `return_scores`, else None).  scores = (Q_h * (1/sqrt(dk))) . K_h^T; where the combined mask
  (query_mask [B, T] & value_mask [B, S] & key_mask [B, S] & the causal triangle s <= t & attention_mask [B, T, S];
  bool / int32 / int64, nonzero = kept) drops a score, -1e9 is added in fp32, as tf-keras's Softmax does.  One launch
  forward, three backward.  Differentiable in Q, K and V; P is returned detached (non-differentiable)."""
  for t, name in ((Q, "query"), (K, "key"), (V, "value")):
    require_cuda(t, name)
    if t.dim() != 3:
      raise ValueError(f"attention: the projected {name} must be [batch, length, heads * dim], got {tuple(t.shape)}")
  H = int(num_heads)
  B, T, S = Q.shape[0], Q.shape[1], K.shape[1]
  if H < 1 or Q.shape[2] % H or V.shape[2] % H:
    raise ValueError(f"attention: {H} heads do not divide the widths {Q.shape[2]} and {V.shape[2]}")
  dk, dv = Q.shape[2] // H, V.shape[2] // H
  if tuple(K.shape) != (B, S, H * dk) or V.shape[:2] != (B, S):
    raise ValueError(f"attention: key {tuple(K.shape)} and value {tuple(V.shape)} do not fit query {tuple(Q.shape)}")
  if T == 0 or S == 0:
    raise ValueError("attention: the query and key sequences must not be empty")
  if not 1 <= dk <= MHA_MAX_HEAD_DIM or not 1 <= dv <= MHA_MAX_HEAD_DIM:
    raise ValueError(f"attention: key_dim = {dk} and value_dim = {dv} must be in 1 .. {MHA_MAX_HEAD_DIM}")
  masks = (_mask_arg(query_mask, (B, T), "attention", "query_mask"),
           _mask_arg(value_mask, (B, S), "attention", "value_mask"),
           _mask_arg(key_mask, (B, S), "attention", "key_mask"),
           _mask_arg(attention_mask, (B, T, S), "attention", "attention_mask"))
  Q, K, V = f32c(Q, "query"), f32c(K, "key"), f32c(V, "value")
  if torch.is_grad_enabled() and any(t.requires_grad for t in (Q, K, V)):
    O, P = _AttentionCore.apply(Q, K, V, H, dk, dv, masks, bool(causal), bool(return_scores))
    return O, (P if return_scores else None)
  O, _, P = _attention_fwd(Q.detach(), K.detach(), V.detach(), H, dk, dv, masks, bool(causal), bool(return_scores),
                           False)
  return O, P


def attention(query: torch.Tensor, value: torch.Tensor, key: Optional[torch.Tensor], query_kernel: torch.Tensor,
              key_kernel: torch.Tensor, value_kernel: torch.Tensor, output_kernel: torch.Tensor, query_bias=None,
              key_bias=None, value_bias=None, output_bias=None, query_mask=None, value_mask=None, key_mask=None,
              attention_mask=None, causal: bool = False, return_scores: bool = False):
  """tf.keras.layers.MultiHeadAttention's call on query [B, T, D_q], value [B, S, D_v] and key [B, S, D_k] (key = value
  when None), with the weights as Keras stores them: query_kernel [D_q, H, dk], key_kernel [D_k, H, dk], value_kernel
  [D_v, H, dv], output_kernel [H, dv, D_out], biases [H, dk] / [H, dk] / [H, dv] / [D_out] (each nullable).  Returns
  (output [B, T, D_out], scores [B, H, T, S] with `return_scores`, else None).  The four projections are K6 Dense calls
  on the kernels viewed as 2-D (no copies); the attention core is K21 (attention_core).  Differentiable in the three
  inputs and all eight weights."""
  key = value if key is None else key
  for t, name in ((query, "query"), (value, "value"), (key, "key")):
    require_cuda(t, name)
    if t.dim() != 3:
      raise NotImplementedError(f"attention: {name} must have rank 3 [batch, length, features], got {tuple(t.shape)}")
  if query_kernel.dim() != 3 or key_kernel.dim() != 3 or value_kernel.dim() != 3 or output_kernel.dim() != 3:
    raise ValueError("attention: the query / key / value / output kernels must be 3-D")
  _, H, dk = query_kernel.shape
  dv = value_kernel.shape[2]
  checks = ((query_kernel, (query.shape[2], H, dk)), (key_kernel, (key.shape[2], H, dk)),
            (value_kernel, (value.shape[2], H, dv)), (output_kernel, (H, dv, output_kernel.shape[2])))
  for w, shape in checks:
    if tuple(w.shape) != tuple(shape):
      raise ValueError(f"attention: a kernel has shape {tuple(w.shape)}, expected {list(shape)}")
  if key.shape[:2] != value.shape[:2] or key.shape[0] != query.shape[0]:
    raise ValueError(f"attention: query {tuple(query.shape)}, value {tuple(value.shape)} and key {tuple(key.shape)} "
                     "must share the batch, and key and value the length")
  B, T, S = query.shape[0], query.shape[1], value.shape[1]
  flat = lambda w, rows: w.reshape(rows, -1)
  vec = lambda b: None if b is None else b.reshape(-1)
  Q = dense(query.reshape(B * T, -1), flat(query_kernel, query.shape[2]), vec(query_bias)).reshape(B, T, H * dk)
  K = dense(key.reshape(B * S, -1), flat(key_kernel, key.shape[2]), vec(key_bias)).reshape(B, S, H * dk)
  V = dense(value.reshape(B * S, -1), flat(value_kernel, value.shape[2]), vec(value_bias)).reshape(B, S, H * dv)
  O, P = attention_core(Q, K, V, H, query_mask, value_mask, key_mask, attention_mask, causal, return_scores)
  out = dense(O.reshape(B * T, H * dv), flat(output_kernel, H * dv), output_bias).reshape(B, T, -1)
  return out, P


# ------------------------------------------------------------------------------------------------
# Dense attention: layers.Attention (K21 dot scores, K25 concat scores) and layers.AdditiveAttention (K25)
# ------------------------------------------------------------------------------------------------
DENSE_SCORE_MODES = {"dot": 0, "concat": 1, "additive": 2}   # TFRS_DENSE_* of include/tfrs_b200.h


class _DenseAttentionDesc(ctypes.Structure):
  _fields_ = [("mode", c_i), ("scale", c_p), ("concat_weight", c_p), ("query_mask", c_p), ("query_mask_kind", c_i),
              ("value_mask", c_p), ("value_mask_kind", c_i), ("causal", c_i), ("rate", _ffi.c_d), ("seed", _ffi.c_u64),
              ("call", _ffi.c_u64)]


def _dense_desc(mode, scale, cw, qm, vm, causal, rate, seed, call) -> _DenseAttentionDesc:
  """qm, vm: the query and value masks as _mask_arg's (mask, kind) pairs."""
  s = _DenseAttentionDesc()
  s.mode, s.scale, s.concat_weight = mode, ptr(scale), ptr(cw)
  s.query_mask, s.query_mask_kind = ptr(qm[0]), qm[1]
  s.value_mask, s.value_mask_kind = ptr(vm[0]), vm[1]
  s.causal, s.rate, s.seed, s.call = int(causal), float(rate), seed, call
  return s


def _dense_attention_fwd(q, k, v, args, want_p, save):
  B, Tq, dim = q.shape
  Tv, dv = v.shape[1], v.shape[2]
  O = torch.empty((B, Tq, dv), dtype=torch.float32, device=q.device)
  stats = torch.empty((B, Tq, 2), dtype=torch.float32, device=q.device) if save else None
  P = torch.empty((B, Tq, Tv), dtype=torch.float32, device=q.device) if want_p else None
  d = _dense_desc(*args)
  check(lib().tfrs_dense_attention_fwd_f32(ptr(q), ptr(k), ptr(v), ctypes.byref(d), B, Tq, Tv, dim, dv, ptr(O),
                                           ptr(stats), ptr(P), stream()), "dense_attention_fwd")
  return O, stats, P


class _DenseAttention(torch.autograd.Function):
  """(O, P or an empty tensor); differentiable in q, k, v, scale and concat_weight.  P is not differentiable."""

  @staticmethod
  def forward(ctx, q, k, v, scale, cw, qm, vm, mode, causal, rate, seed, call, want_p):
    args = (mode, scale, cw, qm, vm, causal, rate, seed, call)
    O, stats, P = _dense_attention_fwd(q, k, v, args, want_p, True)
    P = P if want_p else torch.empty((0,), dtype=torch.float32, device=q.device)
    ctx.save_for_backward(q, k, v, scale, cw, qm[0], vm[0], O, stats)
    ctx.args = (mode, qm[1], vm[1], causal, rate, seed, call)
    ctx.mark_non_differentiable(P)
    ctx.set_materialize_grads(False)
    return O, P

  @staticmethod
  def backward(ctx, dO, _dP):
    q, k, v, scale, cw, qm, vm, O, stats = ctx.saved_tensors
    mode, qk, vk, causal, rate, seed, call = ctx.args
    n = ctx.needs_input_grad
    B, Tq, dim = q.shape
    Tv, dv = v.shape[1], v.shape[2]
    dq, dk, dv_ = torch.empty_like(q), torch.empty_like(k), torch.empty_like(v)
    dscale = torch.empty_like(scale) if n[3] else None
    dcw = torch.empty_like(cw) if n[4] else None
    if dO is None or B == 0:
      for t in (dq, dk, dv_, dscale, dcw):
        if t is not None:
          t.zero_()
    else:
      dO = f32c(dO, "grad")
      d = _dense_desc(mode, scale, cw, (qm, qk), (vm, vk), causal, rate, seed, call)
      ws = workspace(lib().tfrs_dense_attention_bwd_workspace_bytes(mode, B, Tq, dim), q.device, "dense_attention_bwd")
      check(lib().tfrs_dense_attention_bwd_f32(ptr(q), ptr(k), ptr(v), ctypes.byref(d), ptr(O), ptr(stats), ptr(dO), B,
                                               Tq, Tv, dim, dv, ptr(dq), ptr(dk), ptr(dv_), ptr(dscale), ptr(dcw),
                                               ptr(ws), ws.numel(), stream()), "dense_attention_bwd")
    return (dq if n[0] else None, dk if n[1] else None, dv_ if n[2] else None, dscale, dcw) + (None,) * 8


def dense_attention(query: torch.Tensor, key: torch.Tensor, value: torch.Tensor, score_mode: str = "dot", scale=None,
                    concat_weight=None, query_mask=None, value_mask=None, causal: bool = False, rate: float = 0.0,
                    seed: int = 0, call: int = 0, return_scores: bool = False):
  """tf-keras's BaseDenseAttention core on query [B, Tq, dim], key [B, Tv, dim] and value [B, Tv, dv] (float32, CUDA;
  dim, dv <= MHA_MAX_HEAD_DIM) -> (out [B, Tq, dv], weights [B, Tq, Tv] with `return_scores`, else None).  Scores:
  "dot" (q . k) * scale; "concat" concat_weight * sum_d tanh(scale (q_d + k_d)); "additive" sum_d scale_d tanh(q_d +
  k_d); scale None = 1 (a scalar tensor for dot / concat, [dim] for additive).  A score the value mask [B, Tv] or the
  causal triangle drops gets -1e9, then softmax over Tv; with rate > 0 the weights are dropped by Philox4x32-10 at
  (seed, call) as K23 drops a [B, Tq, Tv] tensor and the kept ones scaled by 1 / (1 - rate); out = weights . value,
  zeroed on the rows query_mask [B, Tq] drops.  Masks are bool / int32 / int64, nonzero = kept.  The weights returned
  are the ones value was multiplied by, detached.  One launch forward; three backward plus one fixed-order fold per
  weight gradient.  Differentiable in query, key, value, scale and concat_weight."""
  if score_mode not in DENSE_SCORE_MODES:
    raise ValueError(f"dense_attention: score_mode must be 'dot', 'concat' or 'additive', got {score_mode!r}")
  mode = DENSE_SCORE_MODES[score_mode]
  for t, name in ((query, "query"), (key, "key"), (value, "value")):
    require_cuda(t, name)
    if t.dim() != 3:
      raise ValueError(f"dense_attention: {name} must be [batch, length, dim], got {tuple(t.shape)}")
  B, Tq, dim = query.shape
  Tv, dv = value.shape[1], value.shape[2]
  if tuple(key.shape) != (B, Tv, dim) or value.shape[0] != B:
    raise ValueError(f"dense_attention: key {tuple(key.shape)} and value {tuple(value.shape)} do not fit query "
                     f"{tuple(query.shape)}")
  if Tq == 0 or Tv == 0:
    raise ValueError("dense_attention: the query and value sequences must not be empty")
  if not 1 <= dim <= MHA_MAX_HEAD_DIM or not 1 <= dv <= MHA_MAX_HEAD_DIM:
    raise ValueError(f"dense_attention: dim = {dim} and value dim = {dv} must be in 1 .. {MHA_MAX_HEAD_DIM}, the "
                     "kernels' ceiling")
  if not 0.0 <= float(rate) < 1.0:
    raise ValueError(f"dense_attention: rate must be in [0, 1), got {rate}")
  want = (dim,) if mode == DENSE_SCORE_MODES["additive"] else (1,)
  if scale is not None:
    require_cuda(scale, "scale")
    if scale.numel() != want[0] or (mode == DENSE_SCORE_MODES["additive"] and scale.dim() != 1):
      raise ValueError(f"dense_attention: scale must have {want[0]} element(s), got shape {tuple(scale.shape)}")
    scale = f32c(scale, "scale")
  if mode == DENSE_SCORE_MODES["concat"]:
    if concat_weight is None or concat_weight.numel() != 1:
      raise ValueError("dense_attention: concat scores need a one-element concat_weight")
    require_cuda(concat_weight, "concat_weight")
    concat_weight = f32c(concat_weight, "concat_weight")
  else:
    concat_weight = None
  qm = _mask_arg(query_mask, (B, Tq), "dense_attention", "query_mask")
  vm = _mask_arg(value_mask, (B, Tv), "dense_attention", "value_mask")
  q, k, v = f32c(query, "query"), f32c(key, "key"), f32c(value, "value")
  seed, call = int(seed) & (2**64 - 1), int(call) & (2**64 - 1)
  diff = (q, k, v, scale, concat_weight)
  if torch.is_grad_enabled() and any(t is not None and t.requires_grad for t in diff):
    O, P = _DenseAttention.apply(q, k, v, scale, concat_weight, qm, vm, mode, bool(causal), float(rate), seed, call,
                                 bool(return_scores))
    return O, (P if return_scores else None)
  det = lambda t: None if t is None else t.detach()
  args = (mode, det(scale), det(concat_weight), qm, vm, bool(causal), float(rate), seed, call)
  O, _, P = _dense_attention_fwd(q.detach(), k.detach(), v.detach(), args, bool(return_scores), False)
  return O, P


# ------------------------------------------------------------------------------------------------
# K22 layer normalization: layers.LayerNormalization over the last axis
# ------------------------------------------------------------------------------------------------
def _layer_norm_fwd(x2, gamma, beta, eps, save):
  N, d = x2.shape
  y = torch.empty_like(x2)
  mean = torch.empty((N, 2), dtype=torch.float32, device=x2.device) if save else None    # the pair (hi, lo)
  rstd = torch.empty((N,), dtype=torch.float32, device=x2.device) if save else None
  check(lib().tfrs_layer_norm_fwd_f32(ptr(x2), ptr(gamma), ptr(beta), N, d, float(eps), ptr(y), ptr(mean), ptr(rstd),
                                      stream()), "layer_norm_fwd")
  return y, mean, rstd


class _LayerNorm(torch.autograd.Function):

  @staticmethod
  def forward(ctx, x2, gamma, beta, eps):
    y, mean, rstd = _layer_norm_fwd(x2, gamma, beta, eps, True)
    ctx.save_for_backward(x2, gamma, mean, rstd)
    ctx.set_materialize_grads(False)
    return y

  @staticmethod
  def backward(ctx, dy):
    x2, gamma, mean, rstd = ctx.saved_tensors
    N, d = x2.shape
    n_x, n_g, n_b = ctx.needs_input_grad[:3]
    dx = torch.empty_like(x2) if n_x else None
    dparams = torch.empty((2, d), dtype=torch.float32, device=x2.device) if (n_g or n_b) else None
    if dy is None:
      for t in (dx, dparams):
        if t is not None:
          t.zero_()
    else:
      dy = f32c(dy, "grad")
      ws = workspace(lib().tfrs_layer_norm_bwd_workspace_bytes(N, d), x2.device, "layer_norm_bwd")
      check(lib().tfrs_layer_norm_bwd_f32(ptr(x2), ptr(gamma), ptr(mean), ptr(rstd), ptr(dy), N, d, ptr(dx),
                                          ptr(dparams), ptr(ws), ws.numel(), stream()), "layer_norm_bwd")
    return (dx, dparams[0] if n_g else None, dparams[1] if n_b else None, None)


def layer_norm(x: torch.Tensor, gamma: Optional[torch.Tensor] = None, beta: Optional[torch.Tensor] = None,
               epsilon: float = 1e-3) -> torch.Tensor:
  """tf.keras.layers.LayerNormalization(axis=-1): y = (x - mean) * rsqrt(var + epsilon) * gamma + beta over the last
  axis of x (float32, CUDA), population variance, two passes, the mean kept as an fp32 pair so that x - mean stays exact
  where |mean| >> std; gamma / beta [d] or None (scale / center off).  One K22
  launch forward; the backward is one launch for dx and the per-CTA dgamma / dbeta partials plus a fixed-order fold.
  Differentiable in x, gamma and beta."""
  require_cuda(x, "inputs")
  if x.dim() == 0:
    raise ValueError("layer_norm: the input must have at least one axis")
  d = x.shape[-1]
  if d == 0:
    raise ValueError("layer_norm: the normalized axis is empty")
  for p, name in ((gamma, "gamma"), (beta, "beta")):
    if p is not None and tuple(p.shape) != (d,):
      raise ValueError(f"layer_norm: {name} must be [{d}], got {tuple(p.shape)}")
  x2 = f32c(x, "inputs").reshape(-1, d)
  g = None if gamma is None else f32c(gamma, "gamma")
  b = None if beta is None else f32c(beta, "beta")
  if torch.is_grad_enabled() and any(t is not None and t.requires_grad for t in (x2, g, b)):
    return _LayerNorm.apply(x2, g, b, float(epsilon)).reshape(x.shape)
  y, _, _ = _layer_norm_fwd(x2.detach(), None if g is None else g.detach(), None if b is None else b.detach(), epsilon,
                            False)
  return y.reshape(x.shape)


# ------------------------------------------------------------------------------------------------
# K23 dropout: layers.Dropout / SpatialDropout1D in training, one counter-based Philox kernel both ways
# ------------------------------------------------------------------------------------------------
DROPOUT_MAX_RANK = 4   # TFRS_DROPOUT_MAX_RANK of include/tfrs_b200.h


def dropout_noise_shape(shape, noise_shape) -> Tuple[int, ...]:
  """Keras's noise shape for an input of `shape`: a None entry takes the input's size, and every entry must be 1 (one
  mask value broadcast along that axis) or the input's size."""
  shape = tuple(int(s) for s in shape)
  if noise_shape is None:
    return shape
  if len(noise_shape) != len(shape):
    raise ValueError(f"dropout: noise_shape {tuple(noise_shape)} does not broadcast to the input's shape {shape}")
  noise = tuple(shape[a] if s is None else int(s) for a, s in enumerate(noise_shape))
  if any(n not in (1, s) for n, s in zip(noise, shape)):
    raise ValueError(f"dropout: noise_shape {tuple(noise_shape)} does not broadcast to the input's shape {shape}")
  return noise


def _dropout_launch(x, rate, key, call, noise):
  y = torch.empty_like(x, memory_format=torch.contiguous_format)
  arr = lambda v: ctypes.cast((ctypes.c_int64 * len(v))(*v), c_p)
  check(lib().tfrs_dropout_f32(ptr(x), x.dim(), arr(x.shape), arr(noise), float(rate), key, call, ptr(y), stream()),
        "dropout")
  return y


class _Dropout(torch.autograd.Function):

  @staticmethod
  def forward(ctx, x, rate, key, call, noise):
    ctx.args = (rate, key, call, noise)
    return _dropout_launch(x, rate, key, call, noise)

  @staticmethod
  def backward(ctx, dy):
    return _dropout_launch(f32c(dy, "grad"), *ctx.args), None, None, None, None


def dropout(x: torch.Tensor, rate: float, key: int, call: int, noise_shape=None) -> torch.Tensor:
  """tf.keras.layers.Dropout in training: y = keep ? x * f32(1 / (1 - rate)) : +0 over x (float32, CUDA, rank 1 to
  DROPOUT_MAX_RANK).  The mask is Philox4x32-10 at the 64-bit `key` and the 64-bit counter `call` (include/tfrs_b200.h,
  K23); `noise_shape` follows Keras.  Differentiable in x: the backward regenerates the mask from (key, call), nothing is
  stored.  One launch each way, also at rate 0 (the layers skip that call)."""
  require_cuda(x, "inputs")
  if x.dtype != torch.float32:
    raise TypeError(f"dropout: inputs must be float32, got {x.dtype}")
  if not 1 <= x.dim() <= DROPOUT_MAX_RANK:
    raise NotImplementedError(f"dropout: an input of rank {x.dim()} is not supported (rank 1 to {DROPOUT_MAX_RANK})")
  if not 0.0 <= float(rate) < 1.0:
    raise ValueError(f"dropout: rate must be in [0, 1), got {rate}")
  noise = dropout_noise_shape(x.shape, noise_shape)
  key, call = int(key) & (2**64 - 1), int(call) & (2**64 - 1)
  xc = x.contiguous()
  if torch.is_grad_enabled() and x.requires_grad:
    return _Dropout.apply(xc, float(rate), key, call, noise)
  return _dropout_launch(xc.detach(), float(rate), key, call, noise)


# ------------------------------------------------------------------------------------------------
# K24 batch normalization: layers.BatchNormalization over the last axis
# ------------------------------------------------------------------------------------------------
def _bn_fwd(x2, m, mk, gamma, beta, mm, mv, training, momentum, eps, save):
  N, d = x2.shape
  y = torch.empty_like(x2)
  saved = torch.empty((3 * d + 1,), dtype=torch.float32, device=x2.device) if save else None   # (hi, lo, rstd, n)
  nb = lib().tfrs_batch_norm_fwd_workspace_bytes(N, d) if training else 0
  ws = workspace(nb, x2.device, "batch_norm_fwd") if training else None
  check(lib().tfrs_batch_norm_fwd_f32(ptr(x2), ptr(m), mk, ptr(gamma), ptr(beta), N, d, int(training), float(momentum),
                                      float(eps), ptr(mm), ptr(mv), ptr(y), ptr(saved), ptr(ws),
                                      0 if ws is None else ws.numel(), stream()), "batch_norm_fwd")
  if training:   # the kernel wrote the moving statistics through raw pointers; tell autograd they changed
    torch.autograd.graph.increment_version(mm)
    torch.autograd.graph.increment_version(mv)
  return y, saved


class _BatchNorm(torch.autograd.Function):

  @staticmethod
  def forward(ctx, x2, gamma, beta, m, mk, moving, training, momentum, eps):
    y, saved = _bn_fwd(x2, m, mk, gamma, beta, *moving, training, momentum, eps, True)
    ctx.save_for_backward(x2, gamma, saved, m)
    ctx.mk, ctx.training = mk, training
    ctx.set_materialize_grads(False)
    return y

  @staticmethod
  def backward(ctx, dy):
    x2, gamma, saved, m = ctx.saved_tensors
    N, d = x2.shape
    n_x, n_g, n_b = ctx.needs_input_grad[:3]
    dx = torch.empty_like(x2) if n_x else None
    dparams = torch.empty((2, d), dtype=torch.float32, device=x2.device)
    if dy is None:
      dparams.zero_()
      if dx is not None:
        dx.zero_()
    else:
      dy = f32c(dy, "grad")
      ws = workspace(lib().tfrs_batch_norm_bwd_workspace_bytes(N, d), x2.device, "batch_norm_bwd")
      check(lib().tfrs_batch_norm_bwd_f32(ptr(x2), ptr(m), ctx.mk, ptr(gamma), ptr(saved), ptr(dy), N, d,
                                          int(ctx.training), ptr(dx), ptr(dparams), ptr(ws), ws.numel(), stream()),
            "batch_norm_bwd")
    return (dx, dparams[0] if n_g else None, dparams[1] if n_b else None) + (None,) * 6


def batch_norm(x: torch.Tensor, gamma: Optional[torch.Tensor], beta: Optional[torch.Tensor], moving_mean: torch.Tensor,
               moving_variance: torch.Tensor, training: bool, momentum: float = 0.99, epsilon: float = 1e-3,
               mask: Optional[torch.Tensor] = None) -> torch.Tensor:
  """tf.keras.layers.BatchNormalization(axis=-1) over x (float32, CUDA, rank >= 2; the statistics are per last-axis
  column over all other axes).  In training: the batch mean (an fp32 pair) and population variance, restricted to the
  rows `mask` (x.shape[:-1], bool / int32 / int64, nonzero = kept) keeps; y = (x - mean) rsqrt(var + epsilon) gamma +
  beta; moving_mean / moving_variance (float32 [d], contiguous) are updated in place with decay f32(1 - momentum), also
  under no_grad, and their autograd version counters move as after any in-place update.  At inference: y = (x - moving_mean) rsqrt(moving_variance + epsilon) gamma + beta.  gamma / beta [d]
  or None (scale / center off).  Differentiable in x, gamma and beta in both modes; under no_grad nothing is saved.
  K24: three launches forward in training, one at inference; three backward in training, two at inference."""
  require_cuda(x, "inputs")
  if x.dim() < 2:
    raise ValueError(f"batch_norm: the input must have at least two axes, got {tuple(x.shape)}")
  d = x.shape[-1]
  N = x.numel() // d if d else 0
  if d == 0 or N == 0:
    raise ValueError(f"batch_norm: the input {tuple(x.shape)} is empty")
  for p, name in ((gamma, "gamma"), (beta, "beta"), (moving_mean, "moving_mean"), (moving_variance, "moving_variance")):
    if p is not None and tuple(p.shape) != (d,):
      raise ValueError(f"batch_norm: {name} must be [{d}], got {tuple(p.shape)}")
  for p, name in ((moving_mean, "moving_mean"), (moving_variance, "moving_variance")):
    require_cuda(p, name)
    if p.dtype != torch.float32 or not p.is_contiguous():
      raise TypeError(f"batch_norm: {name} must be a contiguous float32 tensor (it is updated in place)")
  m, mk = _mask_arg(mask, x.shape[:-1], "batch_norm")
  m = None if m is None else m.reshape(N)
  x2 = f32c(x, "inputs").reshape(N, d)
  g = None if gamma is None else f32c(gamma, "gamma")
  b = None if beta is None else f32c(beta, "beta")
  moving = (moving_mean.detach(), moving_variance.detach())
  if torch.is_grad_enabled() and any(t is not None and t.requires_grad for t in (x2, g, b)):
    return _BatchNorm.apply(x2, g, b, m, mk, moving, bool(training), float(momentum), float(epsilon)).reshape(x.shape)
  y, _ = _bn_fwd(x2.detach(), m, mk, None if g is None else g.detach(), None if b is None else b.detach(), *moving,
                 bool(training), momentum, epsilon, False)
  return y.reshape(x.shape)
