"""Embedding lookup with sparse gradients -- the role `tf.keras.layers.Embedding` (+ IndexedSlices
gradients) plays in the reference's user/item towers (README.md:62-66,77-78).

Forward = libtfrs_b200's gather kernel.  Backward does NOT build a dense [rows, dim] gradient: it records
(ids, grad_rows) on the table (the IndexedSlices of TF), which `recommenders_b200.optimizers.Adagrad`
consumes with the deterministic sparse-Adagrad kernel."""
from __future__ import annotations

import math
from typing import Callable, Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch

from ... import ops


class _GatherFn(torch.autograd.Function):

  @staticmethod
  def forward(ctx, anchor, module, ids):
    ctx.module = module
    ctx.ids = ids
    return ops.gather([module.weight], [ids])

  @staticmethod
  def backward(ctx, g):
    ctx.module._sparse_grads.append((ctx.ids, g.contiguous()))
    return None, None, None


class Embedding(torch.nn.Module):
  """`tf.keras.layers.Embedding(input_dim, output_dim, mask_zero=False)`; default init uniform(-0.05, 0.05) like Keras.

  With mask_zero=True, `compute_mask(ids)` is `ids != 0`, and the output carries its mask for a following
  GlobalAveragePooling1D (`ops.attached_mask`; honoured only for that very tensor, unmodified: `_version` + `data_ptr`)."""

  def __init__(self, input_dim: int, output_dim: int, device=None, embeddings_initializer="uniform", mask_zero=False):
    super().__init__()
    device = device or torch.device("cuda", torch.cuda.current_device())
    w = torch.empty((input_dim, output_dim), dtype=torch.float32, device=device)
    if embeddings_initializer == "uniform":
      w.uniform_(-0.05, 0.05)
    elif embeddings_initializer == "zeros":
      w.zero_()
    elif callable(embeddings_initializer):
      w.copy_(embeddings_initializer((input_dim, output_dim), device))
    else:
      raise ValueError(f"Unknown initializer: {embeddings_initializer}")
    # not an nn.Parameter: a dense .grad of a 10M-row table must never exist
    self.register_buffer("weight", w)
    self._sparse_grads: List[Tuple[torch.Tensor, torch.Tensor]] = []
    self._anchor = torch.nn.Parameter(torch.zeros((), device=device))  # keeps the autograd edge alive
    self.input_dim, self.output_dim = input_dim, output_dim
    self.mask_zero = bool(mask_zero)

  def compute_mask(self, ids, mask=None):
    if not self.mask_zero:
      return None
    return ids != 0

  def forward(self, ids: torch.Tensor) -> torch.Tensor:
    if ids.dtype.is_floating_point:  # README feeds float ids from tf.strings.to_number (README.md:50-53)
      ids = ids.to(torch.int32)
    shape = ids.shape
    flat = ids.reshape(-1)
    if torch.is_grad_enabled():
      out = _GatherFn.apply(self._anchor, self, flat)
    else:
      out = ops.gather([self.weight], [flat])
    out = out.reshape(*shape, self.output_dim)
    return ops.attach_mask(out, ids if self.mask_zero else None)     # the ids themselves: nonzero = kept

  def pop_sparse_grads(self):
    g, self._sparse_grads = self._sparse_grads, []
    return g


def gather_concat(tables: Sequence[Embedding], ids: Sequence[torch.Tensor], extra: Optional[torch.Tensor] = None,
                  pad_to: int = 1) -> torch.Tensor:
  """Fused multi-table lookup written straight into the concatenated `[B, sum(dims) (+extra)]` activation
  (the `Concatenate()` before `Cross`, experimental/models/ranking.py:41-46).  Inference-only helper."""
  dims = [t.output_dim for t in tables]
  width = sum(dims) + (extra.shape[1] if extra is not None else 0)
  ld = (width + pad_to - 1) // pad_to * pad_to
  n = ids[0].numel()
  out = torch.zeros((n, ld), dtype=torch.float32, device=tables[0].weight.device) if ld != width else \
      torch.empty((n, ld), dtype=torch.float32, device=tables[0].weight.device)
  ops.gather([t.weight for t in tables], [i.reshape(-1) for i in ids], out=out)
  if extra is not None:
    out[:, sum(dims):width] = extra
  return out


# ---- shared by TPUEmbedding and UnifiedEmbedding (layers/feature_multiplexing) ----

def _default_initializer(dim: int):
  """TableConfig's default: truncated normal, mean 0, std 1/sqrt(dim), cut at two standard deviations."""
  std = 1.0 / math.sqrt(dim)

  def init(shape, device):
    return torch.nn.init.trunc_normal_(torch.empty(shape, device=device), 0.0, std, -2.0 * std, 2.0 * std)
  return init


def _ragged_splits(name: str, splits) -> Tuple[Optional[torch.Tensor], Optional[np.ndarray]]:
  """The row_splits of a ragged (values, row_splits) input: (the CUDA int64 tensor, made contiguous, None) or (None, the
  NumPy integer array as int64, for `_upload`)."""
  if isinstance(splits, torch.Tensor):
    ops.require_cuda(splits, f"row_splits of '{name}'")
    if splits.dtype != torch.int64 or splits.dim() != 1:
      raise TypeError(f"row_splits of '{name}' must be a 1-D int64 tensor")
    return splits.contiguous(), None
  if isinstance(splits, np.ndarray) and splits.dtype.kind in "iu" and splits.ndim == 1:
    return None, splits.astype(np.int64)
  raise TypeError(f"row_splits of '{name}' must be an int64 CUDA tensor or a NumPy integer array")


def _upload(i64: Sequence[np.ndarray], device, data: Sequence[np.ndarray] = ()):
  """The contiguous int64 host arrays and uint8 byte buffers of one call in ONE host-to-device copy, the int64 arrays
  first (8-byte aligned).  Returns (the int64 views, the byte views) on the device, each in order; an empty byte buffer
  gets a one-byte view (a non-NULL pointer)."""
  parts = [a.view(np.uint8) for a in i64] + list(data)
  if not parts:
    return [], []
  dev = torch.from_numpy(np.concatenate(parts)).to(device)
  n64 = sum(a.size for a in i64)
  words, pos, byte_pos = dev[:8 * n64].view(torch.int64), 0, 8 * n64
  ints, bufs = [], []
  for a in i64:
    ints.append(words[pos:pos + a.size]); pos += a.size
  for b in data:
    bufs.append(dev[byte_pos:byte_pos + b.size] if b.size else dev[:1]); byte_pos += b.size
  return ints, bufs


def _per_table(table_of: Sequence[int], counts: Sequence[int], alloc):
  """({table: alloc(table, its values in all)}, each lookup's slice): lookup k (counts[k] values of table table_of[k])
  gets the next consecutive slice of its table's buffer, in lookup order."""
  starts, total = [], {}
  for t, n in zip(table_of, counts):
    starts.append(total.get(t, 0)); total[t] = starts[-1] + n
  bufs = {t: alloc(t, n) for t, n in total.items()}
  return bufs, [bufs[t][s:s + n] for t, s, n in zip(table_of, starts, counts)]


def _sparse_grad_ids(table_of: Sequence[int], counts: Sequence[int], device):
  """The forward half of the (ids, rows) sparse gradient of a multi-lookup call: one int64 id buffer per table and its
  slice for each lookup (see `_per_table`), which the forward kernel fills."""
  return _per_table(table_of, counts, lambda t, n: torch.empty(n, dtype=torch.int64, device=device))


def _record_sparse_grads(tables: Sequence[Embedding], table_of: Sequence[int], counts: Sequence[int],
                         ids: Dict[int, torch.Tensor], write_rows: Callable[[List[torch.Tensor]], None]) -> None:
  """The backward half: one float32 [n, dim] rows buffer per table, sliced as the ids were; `write_rows(slices)` runs
  the backward kernel into the slices, then each table records ONE (ids, rows) pair."""
  rows, slices = _per_table(table_of, counts, lambda t, n: torch.empty((n, tables[t].output_dim), dtype=torch.float32,
                                                                       device=ids[t].device))
  write_rows(slices)
  for t, r in rows.items():
    tables[t]._sparse_grads.append((ids[t], r))


from .tpu_embedding_layer import FeatureConfig, TableConfig, TPUEmbedding  # noqa: E402  (needs the names above)
