"""Unified Embedding (Coleman et al., "Unified Embedding: Battle-Tested Feature Representations for Web-Scale ML
Systems"): mirror of tensorflow_recommenders/layers/feature_multiplexing/unified_embedding.py.

Several features share a few embedding tables.  Every feature is split into `num_chunks` chunks; chunk c of the k-th
added feature looks up `tf.keras.layers.Hashing(num_bins=buckets_per_table, salt=[k, c])` of the feature's values in
the next table of a round-robin cursor, and a feature's output is its chunks concatenated in `sorted()` order of the
chunk names.  Here the tables are `layers.embedding.Embedding` modules, so the optimizers train them from sparse
(ids, rows) gradients, and the hashing, the lookups and the pooling of one call run in the K8 kernels (one launch, two
when a ragged feature is pooled, one for the backward).

Inputs, per feature name:
  - a CUDA int32 / int64 tensor [B, ...] -> [B, ..., width] (hashed as its decimal text, like Hashing on integers);
  - a NumPy array of str / bytes (dtype U, S or object) or a list of str -> the same, looked up on the device after one
    host-to-device copy of every string feature of the call (trailing NUL bytes do not survive NumPy's fixed-width
    string types);
  - a ragged `(values, row_splits)` pair as in `tf.RaggedTensor.from_row_splits` (1-D values of either kind, int64
    row_splits [B+1] as a CUDA tensor or a NumPy array) -> [B, width], each bag pooled by the table combiner
    ("mean" by default, "sum" or "sqrtn"); an empty bag gives zeros.
"""
from __future__ import annotations

from typing import Any, Dict, List, NamedTuple, Tuple

import numpy as np
import torch

from ... import ops
from ..._strings import is_strings as _is_strings, pack_strings as _pack_strings
from ..embedding import Embedding, _default_initializer, _ragged_splits, _record_sparse_grads, _sparse_grad_ids, _upload


class FeatureConfig(NamedTuple):
  """The lookup of one chunk: the table it reads and its name (tf.tpu.experimental.embedding.FeatureConfig's role)."""
  table: str
  name: str


_TABLE_KWARGS = ("initializer", "combiner")


class UnifiedEmbeddingConfig:
  """`num_tables` tables of [buckets_per_table, dim_per_table] named f"{name}_{i}", shared by the features added with
  `add_feature`.  Of the TableConfig arguments, `initializer` (a callable (shape, device) -> tensor, or an
  `Embedding` initializer name) and `combiner` ("mean", "sum", "sqrtn") are accepted."""

  def __init__(self, buckets_per_table: int, dim_per_table: int, num_tables: int, name: str, **kwargs):
    for k in kwargs:
      if k not in _TABLE_KWARGS:
        raise TypeError(f"UnifiedEmbeddingConfig: unsupported table argument '{k}' (accepted: {', '.join(_TABLE_KWARGS)})")
    self._combiner = kwargs.get("combiner", "mean")
    if self._combiner not in ops.COMBINERS:
      raise ValueError(f"combiner must be one of {sorted(ops.COMBINERS)}, got {self._combiner!r}")
    self._initializer = kwargs.get("initializer")
    self._buckets_per_table = buckets_per_table
    self._dim_per_table = dim_per_table
    self._num_tables = num_tables
    self._current_table = 0
    self._num_features = 0
    self._name = name
    self._table_names = [f"{name}_{i}" for i in range(num_tables)]
    self._embed_configs: Dict[str, Dict[str, FeatureConfig]] = {}
    self._hashing_configs: Dict[str, Dict[str, Dict[str, Any]]] = {}
    self._features: List[Tuple[str, int]] = []
    self._chunk_tables: Dict[str, List[int]] = {}

  def add_feature(self, name: str, num_chunks: int, **kwargs):
    """Adds a feature of `num_chunks` chunks (output width num_chunks * dim_per_table).  The table cursor carries on
    from the previous feature."""
    if kwargs:
      raise TypeError(f"add_feature: unsupported feature argument '{next(iter(kwargs))}'")
    if name in self._embed_configs:
      raise ValueError(f"add_feature: feature '{name}' was already added")
    chunk_embed_configs, chunk_hashing_configs, tables = {}, {}, []
    for chunk_id in range(num_chunks):
      chunk_name = f"{self._name}_{name}_lookup_{chunk_id}"
      chunk_embed_configs[chunk_name] = FeatureConfig(table=self._table_names[self._current_table], name=chunk_name)
      chunk_hashing_configs[chunk_name] = {"num_bins": self._buckets_per_table, "salt": [self._num_features, chunk_id]}
      tables.append(self._current_table)
      self._current_table = (self._current_table + 1) % self._num_tables
    self._num_features += 1
    self._embed_configs[name] = chunk_embed_configs
    self._hashing_configs[name] = chunk_hashing_configs
    self._features.append((name, num_chunks))
    self._chunk_tables[name] = tables

  def _lookup_plan(self) -> List[Tuple[str, List[Tuple[int, Tuple[int, int], int]]]]:
    """Per feature in config order, per chunk in chunk order: (table index, SipHash key, column slot), the column slot
    being the rank of the chunk's name in sorted() -- the order the reference concatenates the chunks in."""
    plan = []
    for feat, nc in self._features:
      names = list(self._hashing_configs[feat])
      order = sorted(names)
      plan.append((feat, [(self._chunk_tables[feat][c], ops.salt_key(self._hashing_configs[feat][names[c]]["salt"]),
                           order.index(names[c])) for c in range(nc)]))
    return plan

  @property
  def embedding_config(self):
    return self._embed_configs

  @property
  def hashing_config(self):
    return self._hashing_configs


class _Feature:
  """One feature's input after classification; string data and NumPy row splits wait for the call's single upload."""

  def __init__(self, name: str, x):
    self.row_splits = self.host_splits = self.strings = self.values = None
    if isinstance(x, tuple) and len(x) == 2:
      values, splits = x
      self.row_splits, self.host_splits = _ragged_splits(name, splits)
      self.n_bags = (self.row_splits if self.row_splits is not None else self.host_splits).shape[0] - 1
    else:
      values = x
    if isinstance(values, torch.Tensor):
      if values.dtype not in (torch.int32, torch.int64):
        raise TypeError(f"feature '{name}': integer tensors (int32 / int64) or strings are accepted, got {values.dtype}")
      ops.require_cuda(values, f"feature '{name}'")
      self.values, self.shape = values.contiguous().view(-1), tuple(values.shape)
    elif _is_strings(values):
      data, offsets, self.shape = _pack_strings(values)
      self.strings = (data, offsets)
    else:
      raise TypeError(f"feature '{name}': expected a CUDA integer tensor, strings or a (values, row_splits) pair, "
                      f"got {type(values).__name__}")
    self.pooled = isinstance(x, tuple) and len(x) == 2
    if self.pooled and len(self.shape) != 1:
      raise ValueError(f"feature '{name}': ragged values must be 1-D")
    self.n = int(np.prod(self.shape, dtype=np.int64))


class _UnifiedLookupFn(torch.autograd.Function):

  @staticmethod
  def forward(ctx, layer, inputs, slots, outs, ids, *anchors):
    ops.unified_lookup(inputs, slots)
    # no output on ctx: out -> grad_fn -> ctx -> out is a cycle the collector cannot break once the node has several
    # outputs, and every call's activations would stay alive.  The backward reads the layout from the gradients.
    ctx.layer, ctx.inputs, ctx.ids = layer, inputs, ids
    ctx.slots = [s._replace(out=None) for s in slots]
    return tuple(outs)

  @staticmethod
  def backward(ctx, *grads):
    layer, slots = ctx.layer, ctx.slots
    slot_grads = [grads[s.input].contiguous() for s in slots]
    _record_sparse_grads(layer._tables, layer._slot_tables, [ctx.inputs[s.input].n for s in slots], ctx.ids,
                         lambda rows: ops.unified_lookup_bwd(ctx.inputs, slots, slot_grads, rows))
    return (None,) * (5 + len(layer._tables))


class UnifiedEmbedding(torch.nn.Module):
  """Hashes every chunk of every configured feature, looks it up in its shared table and concatenates each feature's
  chunks.  Returns a list in the order the features were added.  `optimizer` is accepted for signature parity with the
  reference (where it configures the TPU embedding engine) and ignored: the tables are trained by whichever optimizer
  steps the model, from the sparse gradients this layer records."""

  def __init__(self, config: UnifiedEmbeddingConfig, optimizer=None, device=None):
    super().__init__()
    if config._dim_per_table % 4:
      raise ValueError(f"dim_per_table must be a multiple of 4, got {config._dim_per_table}")
    self._config = config
    init = config._initializer if config._initializer is not None else _default_initializer(config._dim_per_table)
    self._tables = torch.nn.ModuleList(
        [Embedding(config._buckets_per_table, config._dim_per_table, device=device, embeddings_initializer=init)
         for _ in range(config._num_tables)])
    self._plan = config._lookup_plan()
    self._slot_tables = [t for _, chunks in self._plan for t, _, _ in chunks]

  def get_config(self) -> Dict[str, Any]:
    c = self._config
    return {"buckets_per_table": c._buckets_per_table, "dim_per_table": c._dim_per_table, "num_tables": c._num_tables,
            "name": c._name, "combiner": c._combiner, "features": [list(f) for f in c._features]}

  @classmethod
  def from_config(cls, config: Dict[str, Any], device=None) -> "UnifiedEmbedding":
    """A layer with the same tables and features (freshly initialised; load the weights with `load_state_dict`)."""
    cfg = UnifiedEmbeddingConfig(config["buckets_per_table"], config["dim_per_table"], config["num_tables"],
                                 config["name"], combiner=config.get("combiner", "mean"))
    for feat, nc in config["features"]:
      cfg.add_feature(feat, nc)
    return cls(cfg, device=device)

  def forward(self, features: Dict[str, Any]) -> List[torch.Tensor]:
    feats = [_Feature(name, features[name]) for name, _ in self._plan]
    dev = self._tables[0].weight.device
    # every string buffer (bytes and offsets) and NumPy row split of the call in one copy
    words, data = _upload([a for f in feats for a in ((f.strings[1] if f.strings else None), f.host_splits)
                           if a is not None], dev, [f.strings[0] for f in feats if f.strings])
    words, data = iter(words), iter(data)
    for f in feats:
      if f.strings:
        f.values = next(data), next(words)
      if f.host_splits is not None:
        f.row_splits = next(words)
    grad = torch.is_grad_enabled()
    dim = self._config._dim_per_table
    slot_feats = [f for f, (_, chunks) in zip(feats, self._plan) for _ in chunks]
    if grad:
      ids, sids = _sparse_grad_ids(self._slot_tables, [f.n for f in slot_feats], dev)
    else:   # K8's pooling reads the bucket ids of pooled slots
      ids, sids = {}, [torch.empty(f.n, dtype=torch.int64, device=dev) if f.pooled else None for f in slot_feats]
    sids = iter(sids)
    inputs, slots, outs = [], [], []
    for k, (f, (_, chunks)) in enumerate(zip(feats, self._plan)):
      values, offsets = f.values if isinstance(f.values, tuple) else (f.values, None)
      inputs.append(ops.LookupInput(values, offsets, f.row_splits, self._config._combiner))
      out = torch.empty((f.n_bags if f.pooled else f.n, len(chunks) * dim), dtype=torch.float32, device=dev)
      outs.append(out)
      for t, key, pos in chunks:
        slots.append(ops.LookupSlot(k, self._tables[t].weight, key, out, pos * dim, next(sids)))
    if grad:
      outs = _UnifiedLookupFn.apply(self, inputs, slots, outs, ids, *[t._anchor for t in self._tables])
    else:
      ops.unified_lookup(inputs, slots)
    return [o if f.pooled else o.reshape(*f.shape, o.shape[1]) for o, f in zip(outs, feats)]
