"""TPUEmbedding: mirror of tensorflow_recommenders/layers/embedding/tpu_embedding_layer.py as it runs off TPU
(`TPUEmbeddingForServing`: plain table variables trained by the model's optimizer).

A `FeatureConfig` / `TableConfig` structure describes the categorical features; tables are shared by `TableConfig`
identity.  One call looks up every feature in one K11 launch (csrc/embedding_bag.cu) and, under autograd, one backward
launch that hands each table a single (ids, rows) sparse gradient.  The tables are `layers.embedding.Embedding`
modules, so every optimizer of the package trains them.

Inputs, per feature (weights, when given, follow the feature's values):
  - a CUDA int tensor [B] or [B, n] -> [B, dim] or [B, n, dim], each id looked up on its own (no weights);
  - a ragged `(values, row_splits)` pair (1-D CUDA int values, int64 row_splits [B+1] as a CUDA tensor or a NumPy
    array) or a coalesced 2-D `torch.sparse_coo_tensor` [B, n] -> [B, dim] pooled with the table's combiner, or
    [B, L, dim] for a feature with max_sequence_length L > 0 (longer bags cut, shorter ones padded with zeros).
Ids outside [0, vocabulary_size) are dropped with their weights (safe_embedding_lookup_sparse)."""
from __future__ import annotations

from typing import Any, Dict, List, Optional

import torch

from ... import ops
from . import Embedding, _default_initializer, _ragged_splits, _record_sparse_grads, _sparse_grad_ids, _upload


class TableConfig:
  """Stand-in for tf.tpu.experimental.embedding.TableConfig.  `initializer` is a callable (shape, device) -> tensor or
  an `Embedding` initializer name; None is TF's default truncated normal (std 1/sqrt(dim)).  `optimizer` is accepted and
  unused: the model's optimizer trains every table."""

  def __init__(self, vocabulary_size: int, dim: int, initializer=None, optimizer=None, combiner: str = "mean",
               name: Optional[str] = None, quantization_config=None, layout=None):
    if not isinstance(vocabulary_size, int) or vocabulary_size < 1:
      raise ValueError(f"vocabulary_size must be a positive int, got {vocabulary_size!r}")
    if not isinstance(dim, int) or dim < 1:
      raise ValueError(f"dim must be a positive int, got {dim!r}")
    if combiner not in ops.COMBINERS:
      raise ValueError(f"combiner must be one of {sorted(ops.COMBINERS)}, got {combiner!r}")
    if quantization_config is not None:
      raise NotImplementedError("TableConfig: quantization_config is not supported")
    if layout is not None:
      raise NotImplementedError("TableConfig: layout is not supported")
    self.vocabulary_size, self.dim = vocabulary_size, dim
    self.initializer, self.optimizer, self.combiner, self.name = initializer, optimizer, combiner, name

  def __repr__(self):
    return (f"TableConfig(vocabulary_size={self.vocabulary_size}, dim={self.dim}, combiner={self.combiner!r}, "
            f"name={self.name!r})")


class FeatureConfig:
  """Stand-in for tf.tpu.experimental.embedding.FeatureConfig."""

  def __init__(self, table: TableConfig, max_sequence_length: int = 0, validate_weights_and_indices: bool = True,
               output_shape=None, name: Optional[str] = None):
    if not isinstance(table, TableConfig):
      raise ValueError(f"table must be a TableConfig, got {type(table).__name__}")
    if not isinstance(max_sequence_length, int) or max_sequence_length < 0:
      raise ValueError(f"max_sequence_length must be a non-negative int, got {max_sequence_length!r}")
    if output_shape is not None:
      raise NotImplementedError("FeatureConfig: output_shape is not supported")
    self.table, self.max_sequence_length, self.name = table, max_sequence_length, name

  def __repr__(self):
    return f"FeatureConfig(table={self.table!r}, max_sequence_length={self.max_sequence_length}, name={self.name!r})"


def flatten(structure) -> List[Any]:
  """The leaves of nested dicts (sorted keys, as tf.nest), lists and tuples, in order."""
  if isinstance(structure, dict):
    return [x for k in sorted(structure) for x in flatten(structure[k])]
  if isinstance(structure, (list, tuple)):
    return [x for s in structure for x in flatten(s)]
  return [structure]


def flatten_up_to(shallow, structure) -> List[Any]:
  """The subtrees of `structure` at the leaves of `shallow` (tf.nest.flatten_up_to): a ragged (values, row_splits)
  pair stays one input.  A missing subtree (None) gives None for each of its leaves."""
  if structure is None:
    return [None] * len(flatten(shallow))
  if isinstance(shallow, dict):
    if not isinstance(structure, dict) or set(structure) != set(shallow):
      raise ValueError(f"expected a dict with keys {sorted(shallow)}")
    return [x for k in sorted(shallow) for x in flatten_up_to(shallow[k], structure[k])]
  if isinstance(shallow, (list, tuple)):
    if not isinstance(structure, (list, tuple)) or len(structure) != len(shallow):
      raise ValueError(f"expected a list or tuple of {len(shallow)} entries")
    return [x for a, b in zip(shallow, structure) for x in flatten_up_to(a, b)]
  return [structure]


def pack_as(structure, leaves: List[Any]):
  """`leaves` in the nesting of `structure` (the inverse of flatten)."""
  it = iter(leaves)

  def rec(s):
    if isinstance(s, dict):
      vals = {k: rec(s[k]) for k in sorted(s)}
      return {k: vals[k] for k in s}
    if isinstance(s, (list, tuple)):
      return type(s)(rec(x) for x in s)
    return next(it)
  return rec(structure)


class _Input:
  """One feature's input after classification: flat CUDA ids, int64 row splits (None: dense), weights, output shape."""

  def __init__(self, name: str, x, w, seq_len: int):
    self.host_splits = self.row_splits = self.weights = None
    if isinstance(x, torch.Tensor) and x.is_sparse:
      if x.dim() != 2 or not x.is_coalesced():
        raise ValueError(f"feature '{name}': sparse inputs must be coalesced 2-D tensors [batch, n]")
      ops.require_cuda(x, f"feature '{name}'")
      rows = x.indices()[0]
      self.row_splits = torch.searchsorted(rows, torch.arange(x.shape[0] + 1, device=rows.device))
      self.values = x.values()
      if w is not None:
        if not (isinstance(w, torch.Tensor) and w.is_sparse and w._nnz() == x._nnz()):
          raise ValueError(f"weights of '{name}' must be a sparse tensor with the feature's indices")
        w = w.coalesce().values()
    elif isinstance(x, tuple) and len(x) == 2:
      self.values, splits = x
      self.row_splits, self.host_splits = _ragged_splits(name, splits)
      if isinstance(w, tuple):
        w = w[0]
      if isinstance(self.values, torch.Tensor) and self.values.dim() != 1:
        raise ValueError(f"feature '{name}': ragged values must be 1-D")
    elif isinstance(x, torch.Tensor):
      if w is not None:
        raise ValueError(f"feature '{name}': weights are only supported with sparse or ragged inputs")
      self.values = x
    else:
      raise TypeError(f"feature '{name}': expected a CUDA int tensor, a sparse tensor or a (values, row_splits) pair, "
                      f"got {type(x).__name__}")
    if not isinstance(self.values, torch.Tensor) or self.values.dtype not in (torch.int32, torch.int64):
      raise TypeError(f"feature '{name}': ids must be int32 / int64 tensors")
    ops.require_cuda(self.values, f"feature '{name}'")
    self.shape = tuple(self.values.shape)
    self.values = self.values.contiguous().view(-1)
    if w is not None:
      if not isinstance(w, torch.Tensor) or w.numel() != self.values.numel():
        raise ValueError(f"weights of '{name}' must have one entry per value")
      self.weights = ops.require_cuda(w, f"weights of '{name}'").to(torch.float32).contiguous().view(-1)
    self.bagged = self.row_splits is not None or self.host_splits is not None
    self.seq_len = seq_len if self.bagged else 0

  @property
  def n_bags(self) -> int:
    s = self.row_splits if self.row_splits is not None else self.host_splits
    return s.shape[0] - 1


class _BagFn(torch.autograd.Function):

  @staticmethod
  def forward(ctx, tables, feats, table_of, ids, *anchors):
    ops.embedding_bag(feats)
    # no output on ctx (out -> grad_fn -> ctx -> out would keep every call's activations alive); the backward takes the
    # layout from the gradients
    ctx.tables, ctx.table_of, ctx.ids = tables, table_of, ids
    ctx.feats = [f._replace(out=None, ids=None) for f in feats]
    ctx.out_shapes = [f.out.shape for f in feats]
    return tuple(f.out for f in feats)

  @staticmethod
  def backward(ctx, *grads):
    gs = [g.contiguous() if g is not None else torch.zeros(shape, dtype=torch.float32, device=f.values.device)
          for f, g, shape in zip(ctx.feats, grads, ctx.out_shapes)]
    _record_sparse_grads(ctx.tables, ctx.table_of, [f.values.numel() for f in ctx.feats], ctx.ids,
                         lambda rows: ops.embedding_bag_bwd(ctx.feats, gs, rows))
    return (None,) * (4 + len(ctx.tables))


class TPUEmbedding(torch.nn.Module):
  """`TPUEmbedding(feature_config, optimizer, pipeline_execution_with_tensor_core=False, batch_size=None,
  embedding_feature=None)`.  `feature_config` is any nesting of dicts, lists and tuples of FeatureConfig; `call` takes
  the features (and optional weights) in the same nesting and returns the activations in it.  `optimizer`,
  `pipeline_execution_with_tensor_core`, `batch_size` and `embedding_feature` are accepted for signature parity and
  unused: the tables are trained by whichever optimizer steps the model, from the sparse gradients this layer records."""

  def __init__(self, feature_config, optimizer=None, pipeline_execution_with_tensor_core: bool = False,
               batch_size: Optional[int] = None, embedding_feature=None, device=None):
    super().__init__()
    self._feature_config = feature_config
    self._features = flatten(feature_config)
    for f in self._features:
      if not isinstance(f, FeatureConfig):
        raise ValueError(f"feature_config leaves must be FeatureConfig, got {type(f).__name__}")
    self.optimizer = optimizer
    self.pipeline_execution_with_tensor_core = pipeline_execution_with_tensor_core
    self.batch_size = batch_size
    configs: List[TableConfig] = []
    for f in self._features:
      if not any(f.table is c for c in configs):
        configs.append(f.table)
    self._table_configs = configs
    self._tables = torch.nn.ModuleList([
        Embedding(c.vocabulary_size, c.dim, device=device,
                  embeddings_initializer=c.initializer if c.initializer is not None else _default_initializer(c.dim))
        for c in configs])
    self._table_of = [next(i for i, c in enumerate(configs) if f.table is c) for f in self._features]

  @property
  def embedding_tables(self) -> Dict[TableConfig, Embedding]:
    """Each TableConfig (by identity) and its table."""
    return {c: t for c, t in zip(self._table_configs, self._tables)}

  @property
  def serving_config(self):
    raise NotImplementedError("TPUEmbedding.serving_config is not supported")

  def forward(self, features, weights=None) -> Any:
    flat = flatten_up_to(self._feature_config, features)
    flat_w = flatten_up_to(self._feature_config, weights)
    names = [f.name or str(i) for i, f in enumerate(self._features)]
    inputs = [_Input(nm, x, w, fc.max_sequence_length) for nm, x, w, fc in zip(names, flat, flat_w, self._features)]
    dev = self._tables[0].weight.device
    host = [x for x in inputs if x.host_splits is not None]       # every NumPy row split of the call in one copy
    for x, splits in zip(host, _upload([x.host_splits for x in host], dev)[0]):
      x.row_splits = splits
    grad = torch.is_grad_enabled()
    ids, sids = (_sparse_grad_ids(self._table_of, [x.values.numel() for x in inputs], dev) if grad
                 else ({}, [None] * len(inputs)))
    feats = []
    for x, t, sid in zip(inputs, self._table_of, sids):
      cfg = self._table_configs[t]
      f = ops.BagFeature(self._tables[t].weight, x.values, None, x.row_splits, x.weights, cfg.combiner, x.seq_len)
      out = torch.empty((ops.bag_out_rows(f), cfg.dim), dtype=torch.float32, device=dev)
      denom = None
      if grad and x.bagged and x.seq_len == 0 and cfg.combiner != "sum":
        denom = torch.empty(x.n_bags, dtype=torch.float32, device=dev)
      feats.append(f._replace(out=out, ids=sid, denom=denom))
    if grad:
      outs = _BagFn.apply(list(self._tables), feats, self._table_of, ids, *[t._anchor for t in self._tables])
    else:
      ops.embedding_bag(feats)
      outs = [f.out for f in feats]
    shaped = []
    for o, x in zip(outs, inputs):
      if not x.bagged:
        shaped.append(o.reshape(*x.shape, o.shape[1]))
      elif x.seq_len > 0:
        shaped.append(o.reshape(x.n_bags, x.seq_len, o.shape[1]))
      else:
        shaped.append(o)
    return pack_as(self._feature_config, shaped)
