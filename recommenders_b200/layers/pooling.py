"""`GlobalAveragePooling1D`, the layer that turns the reference's title-token embeddings into one vector per title
(`TextVectorization -> Embedding(..., mask_zero=True) -> GlobalAveragePooling1D()`).  K17's masked mean pool, forward and
backward; DESIGN.md §2 (A21) pins its rule."""
from __future__ import annotations

from typing import Any, Dict

import torch

from .. import ops


class GlobalAveragePooling1D(torch.nn.Module):
  """`tf.keras.layers.GlobalAveragePooling1D(keepdims=False)`: [B, T, d] float32 -> [B, d] (or [B, 1, d]).  With a mask
  ([B, T] bool or int ids, nonzero = kept; passed as `mask=` or carried by an `Embedding(mask_zero=True)` output) the
  mean covers the kept positions only, and an all-masked row is 0/0 = NaN, as in Keras.  The gradient reaches the
  embedding's (ids, rows) pairs with zero rows at masked positions."""

  def __init__(self, data_format="channels_last", keepdims=False, name=None):
    super().__init__()
    if data_format == "channels_first":
      raise NotImplementedError("data_format='channels_first' is not supported")
    if data_format != "channels_last":
      raise ValueError(f"Unknown data_format {data_format!r}; expected 'channels_last' or 'channels_first'")
    self.data_format, self.keepdims, self.name = data_format, bool(keepdims), name

  def forward(self, inputs: torch.Tensor, mask=None) -> torch.Tensor:
    out = ops.mean_pool(inputs, ops.layer_mask(inputs, mask))
    return out.unsqueeze(1) if self.keepdims else out

  def get_config(self) -> Dict[str, Any]:
    return {"name": self.name, "data_format": self.data_format, "keepdims": self.keepdims}

  @classmethod
  def from_config(cls, config: Dict[str, Any]):
    return cls(**config)
