"""Embedding lookup with sparse gradients -- the role `tf.keras.layers.Embedding` (+ IndexedSlices
gradients) plays in the reference's user/item towers (README.md:62-66,77-78).

Forward = libtfrs_b200's gather kernel.  Backward does NOT build a dense [rows, dim] gradient: it records
(ids, grad_rows) on the table (the IndexedSlices of TF), which `recommenders_b200.optimizers.Adagrad`
consumes with the deterministic sparse-Adagrad kernel."""
from __future__ import annotations

from typing import List, Optional, Sequence, Tuple

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
    if self.mask_zero:
      out._tfrs_mask = (ids, out._version, out.data_ptr())     # the ids themselves: nonzero = kept
    return out

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


from .tpu_embedding_layer import FeatureConfig, TableConfig, TPUEmbedding  # noqa: E402  (needs Embedding above)
