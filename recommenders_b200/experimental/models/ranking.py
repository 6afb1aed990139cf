"""A configurable DLRM / DCN ranking model: mirror of tensorflow_recommenders/experimental/models/ranking.py:27-257."""
from __future__ import annotations

from typing import Dict, List, Optional

import torch

from ... import losses, metrics, models, tasks
from ...layers import blocks
from ...layers.embedding import Embedding
from ...layers.feature_interaction import DotInteraction


class Ranking(models.Model):
  """Bottom MLP on the dense features, feature interaction with the sparse embeddings, top MLP, ranking task.

  Defaults as in the reference: bottom `MLP([256, 64, 16], final_activation="relu")`, `DotInteraction()`, top
  `MLP([512, 256, 1], final_activation="sigmoid")`, and `tasks.Ranking(BinaryCrossentropy(reduction=NONE))` with AUC
  ("auc"), BinaryAccuracy ("accuracy"), prediction and label means.  `embedding_layer` maps the sparse-feature dict to a
  dict of [B, d] tensors; a `torch.nn.ModuleDict` of `Embedding` (one per feature name) is applied key by key."""

  def __init__(self, embedding_layer: torch.nn.Module, bottom_stack: Optional[torch.nn.Module] = None,
               feature_interaction: Optional[torch.nn.Module] = None, top_stack: Optional[torch.nn.Module] = None,
               concat_dense: bool = True, task: Optional[tasks.Task] = None) -> None:
    super().__init__()
    self._embedding_layer = embedding_layer
    self._concat_dense = concat_dense
    self._bottom_stack = bottom_stack if bottom_stack is not None else blocks.MLP(units=[256, 64, 16], final_activation="relu")
    self._top_stack = top_stack if top_stack is not None else blocks.MLP(units=[512, 256, 1], final_activation="sigmoid")
    self._feature_interaction = feature_interaction if feature_interaction is not None else DotInteraction()
    if task is not None:
      self._task = task
    else:
      self._task = tasks.Ranking(
          loss=losses.BinaryCrossentropy(reduction=losses.Reduction.NONE),
          metrics=[metrics.AUC(name="auc"), metrics.BinaryAccuracy(name="accuracy")],
          prediction_metrics=[metrics.Mean("prediction_mean")],
          label_metrics=[metrics.Mean("label_mean")])

  def compute_loss(self, inputs, training: bool = False) -> torch.Tensor:
    """Loss of ({"dense_features", "sparse_features"}, labels[, sample_weight]) (ranking.py:141-200)."""
    if len(inputs) == 2:
      features, labels = inputs
      sample_weight = None
    elif len(inputs) == 3:
      features, labels, sample_weight = inputs
    else:
      raise ValueError(
          "Inputs should be either a tuple of (features, labels), "
          "or a tuple of (features, labels, sample weights). "
          "Got a length {len(inputs)} tuple instead: {inputs}."
      )
    outputs = self(features, training=training)
    loss = self._task(labels, outputs, sample_weight=sample_weight)
    loss = loss.mean()
    # The reference divides by tf.distribute's num_replicas_in_sync; this model trains on one replica, so that is 1.
    return loss / 1

  def _embed(self, sparse_features: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
    if isinstance(self._embedding_layer, torch.nn.ModuleDict):
      return {k: self._embedding_layer[k](v) for k, v in sparse_features.items()}
    return self._embedding_layer(sparse_features)

  def call(self, inputs: Dict[str, torch.Tensor]) -> torch.Tensor:
    """Prediction [B] of a feature dict (ranking.py:202-237)."""
    dense_features = inputs["dense_features"]
    sparse_features = inputs["sparse_features"]
    sparse_embeddings = self._embed(sparse_features)
    # tf.nest.flatten orders a dict by key; tf.squeeze drops the size-1 axes after the batch axis
    flat = [sparse_embeddings[k] for k in sorted(sparse_embeddings)] if isinstance(sparse_embeddings, dict) \
        else list(sparse_embeddings)
    sparse_embedding_vecs = [v.reshape(v.shape[0], -1) for v in flat]
    dense_embedding_vec = self._bottom_stack(dense_features)
    interaction_args = sparse_embedding_vecs + [dense_embedding_vec]
    interaction_output = self._feature_interaction(interaction_args)
    if self._concat_dense:
      feature_interaction_output = torch.cat([dense_embedding_vec, interaction_output], dim=1)
    else:
      feature_interaction_output = interaction_output
    prediction = self._top_stack(feature_interaction_output)
    return prediction.reshape(-1)

  def forward(self, inputs, training: bool = False):
    return self.call(inputs)

  @property
  def embedding_trainable_variables(self) -> List[torch.Tensor]:
    """The embedding tables (updated by the sparse optimizer path) and any trainable parameter of the embedding layer."""
    tables = [m.weight for m in self._embedding_layer.modules() if isinstance(m, Embedding)]
    anchors = {id(m._anchor) for m in self._embedding_layer.modules() if isinstance(m, Embedding)}
    return tables + [p for p in self._embedding_layer.parameters() if p.requires_grad and id(p) not in anchors]

  @property
  def dense_trainable_variables(self) -> List[torch.nn.Parameter]:
    """All trainable variables that are not embeddings."""
    emb = {id(p) for p in self._embedding_layer.parameters()}
    return [p for p in self.parameters() if p.requires_grad and id(p) not in emb]
