"""Vocabulary lookups: `StringLookup` and `IntegerLookup`, the tf-keras 2.x preprocessing layers that start the reference's
towers (`Sequential([StringLookup(vocabulary=ids, mask_token=None), Embedding(len(ids) + 1, d)])`).

Index layout (tf-keras index_lookup.py; DESIGN.md §2, A20), with m = 1 when `mask_token` is not None (else 0), o =
`num_oov_indices` and V the vocabulary length: the mask token maps to 0, a value outside the vocabulary to m, and
vocabulary[i] to m + o + i; `vocabulary_size()` is m + o + V.  The lookup runs on the device, in one K15 launch per call
(a hash table built once per vocabulary).  Only `output_mode="int"` and `num_oov_indices` 0 or 1 are offered.

Deviations: an entry of the vocabulary equal to the mask or OOV token raises ValueError (tf-keras accepts those tokens at
the head of the list and strips them), and strings lose trailing NUL bytes (NumPy's fixed-width string types drop them).
"""
from __future__ import annotations

from typing import Any, Dict, List, Optional

import numpy as np
import torch

from .. import ops
from .._strings import pack_strings, upload_packed
from ..data import Dataset

_OTHER_OUTPUT_MODES = ("one_hot", "multi_hot", "count", "tf_idf")


def _device() -> torch.device:
  return torch.device("cuda", torch.cuda.current_device())


class _IndexLookup(torch.nn.Module):
  """The rules both layers share; subclasses say how a value becomes a key and how keys go to the device."""

  def __init__(self, max_tokens, num_oov_indices, mask_token, oov_token, vocabulary, invert, output_mode, sparse,
               pad_to_max_tokens, idf_weights, name):
    super().__init__()
    if output_mode != "int":
      if output_mode in _OTHER_OUTPUT_MODES:
        raise NotImplementedError(f"output_mode={output_mode!r} is not supported; only 'int' is")
      raise ValueError(f"Unknown output_mode {output_mode!r}; expected one of {('int',) + _OTHER_OUTPUT_MODES}")
    if sparse:
      raise NotImplementedError("sparse=True is not supported")
    if pad_to_max_tokens:
      raise NotImplementedError("pad_to_max_tokens=True is not supported")
    if idf_weights is not None:
      raise NotImplementedError("idf_weights are not supported (they only apply to output_mode='tf_idf')")
    if isinstance(num_oov_indices, bool) or not isinstance(num_oov_indices, (int, np.integer)):
      raise ValueError(f"num_oov_indices must be an int, got {num_oov_indices!r}")
    if num_oov_indices < 0:
      raise ValueError(f"num_oov_indices must be >= 0, got {num_oov_indices}")
    if num_oov_indices > 1:
      raise NotImplementedError("num_oov_indices > 1 is not supported: tf-keras spreads OOV values over the buckets by "
                                "a hash this project does not restate")
    if max_tokens is not None and max_tokens <= 1:
      raise ValueError(f"max_tokens must be greater than 1 (or None), got {max_tokens}")
    self.max_tokens = max_tokens
    self.num_oov_indices = int(num_oov_indices)
    self.mask_token = mask_token
    self.oov_token = oov_token
    self.invert = bool(invert)
    self.output_mode = output_mode
    self.name = name
    self._vocab = self._empty_vocabulary()
    self._table: Optional[ops.LookupTable] = None
    if vocabulary is not None:
      self.set_vocabulary(vocabulary)

  # -- vocabulary ------------------------------------------------------------------------------------------------------
  @property
  def _m(self) -> int:
    return 0 if self.mask_token is None else 1

  def _base(self) -> int:
    return self._m + self.num_oov_indices

  def vocabulary_size(self) -> int:
    return self._base() + len(self._vocab)

  def get_vocabulary(self, include_special_tokens: bool = True) -> List[Any]:
    words = self._vocab.tolist()
    if not include_special_tokens:
      return words
    return ([self._special(self.mask_token)] if self._m else []) + [self._special(self.oov_token)] * self.num_oov_indices \
        + words

  def set_vocabulary(self, vocabulary, idf_weights=None) -> None:
    """Sets the vocabulary (a list, a NumPy array, or for IntegerLookup a CUDA integer tensor) and builds its table on the
    current device when one is available (otherwise at the first call).  Duplicates, an entry equal to the mask or OOV
    token, and more than max_tokens indices raise ValueError."""
    if idf_weights is not None:
      raise NotImplementedError("idf_weights are not supported (they only apply to output_mode='tf_idf')")
    if isinstance(vocabulary, str):
      raise NotImplementedError("vocabulary files are not supported; pass the vocabulary as a list or an array")
    vocab, device_keys = self._host_vocabulary(vocabulary)
    for what, tok in (("mask_token", self.mask_token), ("oov_token", self.oov_token)):
      if tok is not None and len(vocab) and self._contains(vocab, tok):
        raise ValueError(f"The vocabulary contains the {what} {tok!r}; pass a vocabulary without the special tokens")
    if self.max_tokens is not None and self._base() + len(vocab) > self.max_tokens:
      raise ValueError(f"Attempted to set a vocabulary larger than the maximum vocab size. Received vocabulary size "
                       f"{self._base() + len(vocab)} (including special tokens), max_tokens {self.max_tokens}")
    self._vocab, self._table = vocab, None
    if torch.cuda.is_available():
      self._build(_device(), device_keys)

  def adapt(self, data, batch_size=None, steps=None) -> None:
    """The vocabulary from `data` (an array, a list, or a `data.Dataset` of batches): the distinct values other than the
    mask and OOV tokens, by count descending with ties in ascending order (numeric for ints, bytewise for strings), cut
    to max_tokens minus the special indices."""
    if isinstance(data, Dataset):
      parts = [self._adapt_values(el) for el in data]
    else:
      parts = [self._adapt_values(data)]
    values = np.concatenate(parts) if parts else self._empty_vocabulary()
    for tok in (self.mask_token, self.oov_token):
      if tok is not None and values.size:
        values = values[~self._equal(values, tok)]
    uniq, counts = np.unique(values, return_counts=True)
    order = np.argsort(-counts, kind="stable")
    vocab = uniq[order]
    if self.max_tokens is not None:
      vocab = vocab[:max(self.max_tokens - self._base(), 0)]
    self.set_vocabulary(vocab)

  # -- calls -----------------------------------------------------------------------------------------------------------
  def forward(self, inputs):
    if isinstance(inputs, tuple) and len(inputs) == 2:
      raise NotImplementedError("ragged (values, row_splits) inputs are not supported")
    return self._inverse(inputs) if self.invert else self._lookup(inputs)

  def _table_on(self, device) -> ops.LookupTable:
    if self._table is None or self._table.slots.device != device:
      self._build(device, None)
    return self._table

  def _index_input(self, inputs) -> torch.Tensor:
    """Indices for invert=True: a CUDA int32 / int64 tensor, or NumPy ints uploaded once."""
    if isinstance(inputs, torch.Tensor):
      ops.require_cuda(inputs, "indices")
      if inputs.dtype not in (torch.int32, torch.int64):
        raise TypeError(f"indices must be int32 or int64, got {inputs.dtype}")
      return inputs
    a = np.asarray(inputs)
    if a.size and a.dtype.kind not in "iu":
      raise TypeError(f"indices must be integers, got dtype {a.dtype}")
    return torch.from_numpy(np.ascontiguousarray(a, np.int64)).to(_device())

  # -- checkpointing: the vocabulary and the config, not the table ----------------------------------------------------
  def get_extra_state(self):
    return {"config": self._layout(), "vocabulary": self._vocab_state()}

  def _vocab_state(self):
    return self._vocab.tolist()

  def set_extra_state(self, state):
    if not state:
      return
    if state.get("config") != self._layout():
      raise ValueError(f"The saved lookup layer has the index layout {state.get('config')}, this one "
                       f"{self._layout()}; construct the layer with the same mask_token, oov_token, num_oov_indices and "
                       "invert to restore it.")
    vocab = state["vocabulary"]
    self.set_vocabulary(vocab.numpy() if isinstance(vocab, torch.Tensor) else vocab)

  def _layout(self) -> Dict[str, Any]:
    return {"mask_token": self.mask_token, "oov_token": self.oov_token, "num_oov_indices": self.num_oov_indices,
            "invert": self.invert}

  def get_config(self) -> Dict[str, Any]:
    return {"name": self.name, "max_tokens": self.max_tokens, "num_oov_indices": self.num_oov_indices,
            "mask_token": self.mask_token, "oov_token": self.oov_token, "vocabulary": self._vocab.tolist(),
            "invert": self.invert, "output_mode": self.output_mode}

  @classmethod
  def from_config(cls, config: Dict[str, Any]):
    return cls(**config)


class IntegerLookup(_IndexLookup):
  """`tf.keras.layers.IntegerLookup`: int64 values -> int64 indices (or back, with invert=True).  Inputs are CUDA int32 /
  int64 tensors of any shape or NumPy ints (uploaded once); outputs are int64 CUDA tensors of the same shape."""

  def __init__(self, max_tokens=None, num_oov_indices=1, mask_token=None, oov_token=-1, vocabulary=None,
               vocabulary_dtype="int64", idf_weights=None, invert=False, output_mode="int", sparse=False,
               pad_to_max_tokens=False, name=None):
    if vocabulary_dtype != "int64":
      raise NotImplementedError(f"vocabulary_dtype={vocabulary_dtype!r} is not supported; only 'int64' is")
    for what, tok in (("mask_token", mask_token), ("oov_token", oov_token)):
      if tok is not None and (isinstance(tok, bool) or not isinstance(tok, (int, np.integer))):
        raise ValueError(f"{what} must be an int or None, got {tok!r}")
    if oov_token is None:
      raise ValueError("oov_token must be an int")
    super().__init__(max_tokens, num_oov_indices, None if mask_token is None else int(mask_token), int(oov_token),
                     vocabulary, invert, output_mode, sparse, pad_to_max_tokens, idf_weights, name)
    self.vocabulary_dtype = vocabulary_dtype

  @staticmethod
  def _empty_vocabulary():
    return np.zeros((0,), np.int64)

  @staticmethod
  def _special(tok):
    return tok

  @staticmethod
  def _equal(values, tok):
    return values == tok

  @staticmethod
  def _contains(vocab, tok):
    return bool((vocab == tok).any())

  @staticmethod
  def _host_vocabulary(vocabulary):
    if isinstance(vocabulary, torch.Tensor):
      ops.require_cuda(vocabulary, "vocabulary")
      if vocabulary.dtype not in (torch.int32, torch.int64) or vocabulary.dim() != 1:
        raise TypeError(f"an IntegerLookup vocabulary tensor must be 1-D int32 / int64, got {vocabulary.dtype}")
      keys = vocabulary.to(torch.int64, copy=True).contiguous()     # the table must not see later writes to it
      return keys.cpu().numpy(), keys
    a = np.asarray(vocabulary)
    if a.ndim != 1 or (a.size and a.dtype.kind not in "iu"):
      raise TypeError(f"an IntegerLookup vocabulary must be a 1-D list or array of ints, got dtype {a.dtype}")
    if a.dtype.kind == "u" and a.size and a.max() > np.iinfo(np.int64).max:
      raise ValueError("IntegerLookup vocabulary entries must fit in int64")
    return a.astype(np.int64), None

  def _vocab_state(self):
    return torch.from_numpy(self._vocab.copy())     # a tensor, so torch.load(weights_only=True) restores it

  def _build(self, device, keys) -> None:
    if keys is None or keys.device != device:
      keys = torch.from_numpy(self._vocab).to(device)
    self._table = ops.lookup_build(keys, None, self.mask_token)

  def _adapt_values(self, x) -> np.ndarray:
    a = x.detach().cpu().numpy() if isinstance(x, torch.Tensor) else np.asarray(x)
    if a.size and a.dtype.kind not in "iu":
      raise TypeError(f"IntegerLookup.adapt takes integers, got dtype {a.dtype}")
    return a.reshape(-1).astype(np.int64)

  def _lookup(self, inputs) -> torch.Tensor:
    if isinstance(inputs, torch.Tensor):
      ops.require_cuda(inputs, "inputs")
      if inputs.dtype not in (torch.int32, torch.int64):
        raise TypeError(f"IntegerLookup takes int32 / int64 tensors, got {inputs.dtype}")
      values = inputs
    else:
      try:
        a = np.asarray(inputs)
      except ValueError:
        raise NotImplementedError("ragged inputs are not supported") from None
      if a.dtype == object:
        raise NotImplementedError("ragged inputs are not supported")
      if a.size and a.dtype.kind not in "iu":
        raise TypeError(f"IntegerLookup takes integers, got dtype {a.dtype}")
      values = torch.from_numpy(np.ascontiguousarray(a, np.int64)).to(_device())
    table = self._table_on(values.device)
    return ops.lookup(table, values, self._base(), self._m if self.num_oov_indices else None)

  def _inverse(self, inputs) -> torch.Tensor:
    idx = self._index_input(inputs)
    table = self._table_on(idx.device)
    return ops.lookup_invert(idx, table.size, self._base(), table.keys, self.mask_token, self.oov_token)

  def get_config(self) -> Dict[str, Any]:
    return {**super().get_config(), "vocabulary_dtype": self.vocabulary_dtype}


class StringLookup(_IndexLookup):
  """`tf.keras.layers.StringLookup`: strings -> int64 indices (or back, with invert=True).  Inputs are NumPy str / bytes /
  object arrays or lists of any shape (`str` encoded as UTF-8, so "a" and b"a" are the same value), packed on the host
  and copied to the device once per call; outputs are int64 CUDA tensors of the same shape.  With invert=True, indices
  (CUDA int tensors or NumPy ints) map to a NumPy array of the vocabulary's kind (str or bytes): positions are gathered
  on the device and the strings come from the host copy of the vocabulary."""

  def __init__(self, max_tokens=None, num_oov_indices=1, mask_token=None, oov_token="[UNK]", vocabulary=None,
               idf_weights=None, encoding="utf-8", invert=False, output_mode="int", sparse=False, pad_to_max_tokens=False,
               name=None):
    if str(encoding).lower().replace("-", "").replace("_", "") != "utf8":
      raise NotImplementedError(f"encoding={encoding!r} is not supported; only 'utf-8' is")
    for what, tok in (("mask_token", mask_token), ("oov_token", oov_token)):
      if tok is not None and not isinstance(tok, (str, bytes)):
        raise ValueError(f"{what} must be a str, bytes or None, got {tok!r}")
    if oov_token is None:
      raise ValueError("oov_token must be a string")
    super().__init__(max_tokens, num_oov_indices, mask_token, oov_token, vocabulary, invert, output_mode, sparse,
                     pad_to_max_tokens, idf_weights, name)
    self.encoding = encoding

  @staticmethod
  def _empty_vocabulary():
    return np.zeros((0,), "U1")

  def _special(self, tok):
    """A special token in the vocabulary's kind."""
    if self._vocab.dtype.kind == "S":
      return tok.encode("utf-8") if isinstance(tok, str) else tok
    return tok.decode("utf-8") if isinstance(tok, bytes) else tok

  @staticmethod
  def _as_bytes(tok) -> bytes:
    return tok.encode("utf-8") if isinstance(tok, str) else bytes(tok)

  def _equal(self, values, tok):
    return values == (self._as_bytes(tok) if values.dtype.kind == "S" else self._as_bytes(tok).decode("utf-8"))

  def _contains(self, vocab, tok):
    return bool(self._equal(vocab, tok).any())

  @staticmethod
  def _strings(x) -> np.ndarray:
    if isinstance(x, np.ndarray) and x.dtype.kind in "US":
      return x
    try:
      # lists go through object arrays, so np.asarray cannot turn a number into a string
      a = np.asarray(x, dtype=object) if isinstance(x, (list, tuple)) else np.asarray(x)
    except ValueError:
      raise NotImplementedError("ragged inputs are not supported") from None
    if a.dtype.kind == "O" and a.size:
      kinds = {type(v) for v in a.flat}
      if kinds <= {str, np.str_}:
        a = a.astype("U")
      elif kinds <= {bytes, np.bytes_}:
        a = a.astype("S")
      elif any(isinstance(v, (list, tuple, np.ndarray)) for v in a.flat):
        raise NotImplementedError("ragged inputs are not supported")
      else:
        raise TypeError(f"StringLookup takes str or bytes values, got {sorted(k.__name__ for k in kinds)}")
    if a.size and a.dtype.kind not in "US":
      raise TypeError(f"StringLookup takes str or bytes values, got dtype {a.dtype}")
    return a

  def _host_vocabulary(self, vocabulary):
    if isinstance(vocabulary, torch.Tensor):
      raise TypeError("a StringLookup vocabulary must be a list or a NumPy array of strings")
    a = self._strings(vocabulary)
    if a.ndim != 1:
      raise TypeError(f"a StringLookup vocabulary must be 1-D, got shape {a.shape}")
    return (a if a.size else self._empty_vocabulary()), None

  def _build(self, device, keys) -> None:
    data, offsets, _ = pack_strings(self._vocab)
    mask = None if self.mask_token is None else np.frombuffer(self._as_bytes(self.mask_token), np.uint8)
    byts, offs, mask_d = upload_packed(data, offsets, device, mask if mask is not None else np.zeros(0, np.uint8))
    self._table = ops.lookup_build(byts, offs, None if mask is None else mask_d)

  def _adapt_values(self, x) -> np.ndarray:
    if isinstance(x, torch.Tensor):
      raise TypeError("StringLookup.adapt takes strings, got a tensor")
    return self._strings(x).reshape(-1)

  def _lookup(self, inputs) -> torch.Tensor:
    if isinstance(inputs, torch.Tensor):
      raise TypeError("StringLookup takes NumPy string arrays or lists of strings, got a tensor")
    a = self._strings(inputs)
    if a.size == 0:
      a = np.zeros(a.shape, "S1")
    data, offsets, shape = pack_strings(a)
    dev = _device()
    table = self._table_on(dev)
    byts, offs = upload_packed(data, offsets, dev)
    out = ops.lookup(table, (byts, offs), self._base(), self._m if self.num_oov_indices else None)
    return out.reshape(shape)

  def _inverse(self, inputs) -> np.ndarray:
    idx = self._index_input(inputs)
    table = self._table_on(idx.device)
    V = table.size
    # position codes: p < V for vocabulary[p], V for the mask token, V + 1 for the OOV token
    codes = ops.lookup_invert(idx, V, self._base(), None, V if self._m else None, V + 1)
    mask = self._special(self.mask_token) if self._m else self._special(self.oov_token)
    words = np.concatenate([self._vocab, np.asarray([mask, self._special(self.oov_token)], dtype=self._vocab.dtype.kind)])
    return words[codes.cpu().numpy()]

  def get_config(self) -> Dict[str, Any]:
    return {**super().get_config(), "encoding": self.encoding}
