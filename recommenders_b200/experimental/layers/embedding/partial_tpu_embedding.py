"""PartialTPUEmbedding: mirror of tensorflow_recommenders/experimental/layers/embedding/partial_tpu_embedding.py:26-142.

Tables with vocabulary_size <= size_threshold become plain `layers.embedding.Embedding` lookups (one per TableConfig,
shared by the features that name it; dense inputs only), the larger ones one `TPUEmbedding`.  size_threshold=None puts
every table in an Embedding, 0 (or any negative value) every table in the TPUEmbedding."""
from __future__ import annotations

from typing import Dict, Optional

import torch

from ....layers.embedding import Embedding, TPUEmbedding


class PartialTPUEmbedding(torch.nn.Module):
  """`PartialTPUEmbedding(feature_config, optimizer, pipeline_execution_with_tensor_core=False, batch_size=None,
  size_threshold=10_000)` over a dict of FeatureConfig.  `optimizer`, `pipeline_execution_with_tensor_core` and
  `batch_size` are accepted and unused, as in TPUEmbedding."""

  def __init__(self, feature_config, optimizer=None, pipeline_execution_with_tensor_core: bool = False,
               batch_size: Optional[int] = None, size_threshold: Optional[int] = 10_000, device=None):
    super().__init__()
    tpu_feature_config = {}
    table_to_emb = {}
    self._keras_embedding_layers: Dict[str, Embedding] = {}
    for name, fc in feature_config.items():
      table = fc.table
      if size_threshold is not None and table.vocabulary_size > size_threshold:
        tpu_feature_config[name] = fc
        continue
      if id(table) not in table_to_emb:
        table_to_emb[id(table)] = Embedding(table.vocabulary_size, table.dim, device=device,
                                            embeddings_initializer=table.initializer or "uniform")
      self._keras_embedding_layers[name] = table_to_emb[id(table)]
    # registered once per table, in order of first use
    self._keras_tables = torch.nn.ModuleList(list({id(m): m for m in self._keras_embedding_layers.values()}.values()))
    self._tpu_embedding = TPUEmbedding(tpu_feature_config, optimizer, pipeline_execution_with_tensor_core,
                                       device=device) if tpu_feature_config else None

  def forward(self, inputs: Dict[str, object]) -> Dict[str, torch.Tensor]:
    output = {}
    for key, val in inputs.items():
      if key in self._keras_embedding_layers:
        if not isinstance(val, torch.Tensor) or val.is_sparse:
          raise ValueError("Only dense tensor input is supported for Keras embedding layers, but got: "
                           f"{type(val).__name__}")
        output[key] = self._keras_embedding_layers[key](val)
    if self._tpu_embedding is not None:
      output.update(self._tpu_embedding({k: v for k, v in inputs.items() if k not in self._keras_embedding_layers}))
    return output

  @property
  def tpu_embedding(self) -> Optional[TPUEmbedding]:
    """The TPUEmbedding of the large tables, or None."""
    return self._tpu_embedding

  @property
  def keras_embedding_layers(self) -> Dict[str, Embedding]:
    """Feature name -> the Embedding of its small table."""
    return self._keras_embedding_layers
