"""Vocabulary lookups: `StringLookup` and `IntegerLookup`, the tf-keras 2.x preprocessing layers that start the reference's
towers (`Sequential([StringLookup(vocabulary=ids, mask_token=None), Embedding(len(ids) + 1, d)])`).

Index layout (tf-keras index_lookup.py; DESIGN.md §2, A20), with m = 1 when `mask_token` is not None (else 0), o =
`num_oov_indices` and V the vocabulary length: the mask token maps to 0, a value outside the vocabulary to m, and
vocabulary[i] to m + o + i; `vocabulary_size()` is m + o + V.  The lookup runs on the device, in one K15 launch per call
(a hash table built once per vocabulary).  Only `output_mode="int"` and `num_oov_indices` 0 or 1 are offered.

Deviations: an entry of the vocabulary equal to the mask or OOV token raises ValueError (tf-keras accepts those tokens at
the head of the list and strips them), and strings lose trailing NUL bytes (NumPy's fixed-width string types drop them).

The text and numeric feature layers of the reference's featurization / context_features / deep_recommenders towers
follow: `TextVectorization` (K16, on the table of an inner StringLookup), `Discretization` and `Normalization` (K17);
DESIGN.md §2, A21.  `Hashing` (K18; DESIGN.md §2, A22) is the vocabulary-free alternative to the lookups.
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


# ---------------------------------------------------------------------------------------------------------------------
# Text and numeric feature columns (DESIGN.md §2, A21): TextVectorization (K16), Discretization and Normalization (K17)
# ---------------------------------------------------------------------------------------------------------------------
_STANDARDIZE = {None: 0, "lower": ops.TEXT_LOWER, "strip_punctuation": ops.TEXT_STRIP,
                "lower_and_strip_punctuation": ops.TEXT_LOWER | ops.TEXT_STRIP}
_TEXT_OUTPUT_MODES = ("multi_hot", "count", "tf_idf")


class TextVectorization(torch.nn.Module):
  """`tf.keras.layers.TextVectorization` with output_mode="int" and split="whitespace": strings -> int64 [B, T] token
  indices.  Inputs are NumPy str / bytes / object arrays or lists of shape [B] or [B, 1], packed on the host and copied
  to the device once per call.  The output is an int64 CUDA tensor padded with 0; T is `output_sequence_length` when it
  is given (longer token lists are truncated), else the longest token count of the batch (one 4-byte host read).

  Standardize lowercases ASCII and deletes the 32 ASCII punctuation bytes; the split is on runs of " \\t\\n\\v\\f\\r".
  Index 0 is padding, 1 is OOV, vocabulary entry i is 2 + i.  As in Keras, the vocabulary lives in an inner
  `StringLookup(mask_token="", oov_token="[UNK]")`, whose K15 table the K16 kernels probe: two launches per call."""

  def __init__(self, max_tokens=None, standardize="lower_and_strip_punctuation", split="whitespace", ngrams=None,
               output_mode="int", output_sequence_length=None, pad_to_max_tokens=False, vocabulary=None,
               idf_weights=None, sparse=False, ragged=False, encoding="utf-8", name=None):
    super().__init__()
    if callable(standardize):
      raise NotImplementedError("a callable standardize is not supported")
    if standardize not in _STANDARDIZE:
      raise ValueError(f"Unknown standardize {standardize!r}; expected one of {tuple(_STANDARDIZE)} or a callable")
    if split is None or split == "character" or callable(split):
      raise NotImplementedError(f"split={split!r} is not supported; only 'whitespace' is")
    if split != "whitespace":
      raise ValueError(f"Unknown split {split!r}; expected 'whitespace', 'character', None or a callable")
    if ngrams is not None:
      raise NotImplementedError("ngrams are not supported")
    if output_mode != "int":
      if output_mode in _TEXT_OUTPUT_MODES:
        raise NotImplementedError(f"output_mode={output_mode!r} is not supported; only 'int' is")
      raise ValueError(f"Unknown output_mode {output_mode!r}; expected one of {('int',) + _TEXT_OUTPUT_MODES}")
    if output_sequence_length is not None and (isinstance(output_sequence_length, bool) or
                                               not isinstance(output_sequence_length, (int, np.integer)) or
                                               output_sequence_length < 1):
      raise ValueError(f"output_sequence_length must be a positive int or None, got {output_sequence_length!r}")
    if ragged:
      raise NotImplementedError("ragged=True is not supported")
    if max_tokens is not None and max_tokens < 1:
      raise ValueError(f"max_tokens must be > 1, got {max_tokens}")
    self.standardize, self.split, self.ngrams, self.output_mode = standardize, split, ngrams, output_mode
    self.output_sequence_length = None if output_sequence_length is None else int(output_sequence_length)
    self.ragged, self.name = ragged, name
    self._lookup_layer = StringLookup(max_tokens=max_tokens, num_oov_indices=1, mask_token="", oov_token="[UNK]",
                                      vocabulary=vocabulary, idf_weights=idf_weights, encoding=encoding,
                                      output_mode="int", sparse=sparse, pad_to_max_tokens=pad_to_max_tokens)

  @property
  def _flags(self) -> int:
    return _STANDARDIZE[self.standardize]

  # -- vocabulary: the inner StringLookup's ---------------------------------------------------------------------------
  def get_vocabulary(self, include_special_tokens: bool = True) -> List[Any]:
    return self._lookup_layer.get_vocabulary(include_special_tokens)

  def vocabulary_size(self) -> int:
    return self._lookup_layer.vocabulary_size()

  def set_vocabulary(self, vocabulary, idf_weights=None) -> None:
    self._lookup_layer.set_vocabulary(vocabulary, idf_weights)

  def adapt(self, data, batch_size=None, steps=None) -> None:
    """The vocabulary from `data` (an array, a list, or a `data.Dataset` of strings or batches of strings): every token
    the call would produce, by count descending, ties by token descending bytewise (tf-keras's
    `np.lexsort((tokens, counts))[::-1]`), cut to max_tokens - 2.  The tokens come from the device kernels of a call;
    counting and ordering run on the host."""
    counts: Dict[bytes, int] = {}
    for el in (data if isinstance(data, Dataset) else [data]):
      flat = self._batch(el, adapt=True)
      if flat.size == 0:
        continue
      data_h, offsets, _ = pack_strings(flat)
      byts, offs = upload_packed(data_h, offsets, _device())
      buf, spans = ops.text_tokens(byts, offs, self._flags)
      buf = buf.tobytes()
      for s, n in spans.tolist():
        tok = buf[s:s + n]
        counts[tok] = counts.get(tok, 0) + 1
    vocab = sorted(counts, key=lambda t: (counts[t], t), reverse=True)
    max_tokens = self._lookup_layer.max_tokens
    if max_tokens is not None:
      vocab = vocab[:max(max_tokens - 2, 0)]
    try:
      words = np.asarray([t.decode("utf-8") for t in vocab], dtype=object)
    except UnicodeDecodeError:
      words = np.asarray(vocab, dtype=object)
    self._lookup_layer.set_vocabulary(words if len(vocab) else np.zeros((0,), "U1"))

  # -- calls -----------------------------------------------------------------------------------------------------------
  @staticmethod
  def _batch(inputs, adapt=False) -> np.ndarray:
    if isinstance(inputs, torch.Tensor):
      raise TypeError("TextVectorization takes NumPy string arrays or lists of strings, got a tensor")
    if isinstance(inputs, (str, bytes)):
      inputs = [inputs]
    a = StringLookup._strings(inputs)
    if adapt and a.ndim == 0:
      return a.reshape(1)
    if a.ndim == 2 and a.shape[1] == 1:
      return a.reshape(-1)
    if a.ndim != 1:
      raise ValueError(f"TextVectorization takes inputs of shape [B] or [B, 1], got {a.shape}")
    return a

  def forward(self, inputs) -> torch.Tensor:
    if isinstance(inputs, tuple) and len(inputs) == 2:
      raise NotImplementedError("ragged (values, row_splits) inputs are not supported")
    flat = self._batch(inputs)
    dev = _device()
    T = self.output_sequence_length
    if flat.size == 0:
      return torch.zeros((0, T or 0), dtype=torch.int64, device=dev)
    data, offsets, _ = pack_strings(flat)
    table = self._lookup_layer._table_on(dev)
    byts, offs = upload_packed(data, offsets, dev)
    lk = self._lookup_layer
    return ops.text_vectorize(table, byts, offs, self._flags, T, lk._base(), lk._m)

  # -- checkpointing and config ---------------------------------------------------------------------------------------
  def get_config(self) -> Dict[str, Any]:
    lk = self._lookup_layer
    return {"name": self.name, "max_tokens": lk.max_tokens, "standardize": self.standardize, "split": self.split,
            "ngrams": self.ngrams, "output_mode": self.output_mode,
            "output_sequence_length": self.output_sequence_length, "pad_to_max_tokens": False,
            "vocabulary": lk.get_vocabulary(include_special_tokens=False), "idf_weights": None, "sparse": False,
            "ragged": self.ragged, "encoding": lk.encoding}

  @classmethod
  def from_config(cls, config: Dict[str, Any]):
    return cls(**config)


_DISCRETIZATION_OUTPUT_MODES = ("one_hot", "multi_hot", "count")


def _numeric_input(inputs, what: str) -> torch.Tensor:
  """A CUDA int32 / int64 / float32 / float64 tensor, or NumPy numbers uploaded once (other int / float widths widened)."""
  if isinstance(inputs, torch.Tensor):
    ops.require_cuda(inputs, "inputs")
    return inputs
  a = np.asarray(inputs)
  if a.dtype.kind in "iub":
    a = a if a.dtype in (np.int32, np.int64) else a.astype(np.int64)
  elif a.dtype.kind == "f":
    a = a if a.dtype in (np.float32, np.float64) else a.astype(np.float32)
  else:
    raise TypeError(f"{what} takes numbers, got dtype {a.dtype}")
  return torch.from_numpy(np.ascontiguousarray(a)).to(_device())


class Discretization(torch.nn.Module):
  """`tf.keras.layers.Discretization(bin_boundaries)` with output_mode="int": each value -> the int64 index of its bucket,
  #{i : b_i <= x} over the boundaries rounded once to float32 (TF's Bucketize on the CPU).  Integers are compared after
  rounding to float32, float64 values as doubles; NaN falls in the last bucket.  Inputs are CUDA or NumPy int32 / int64
  / float32 / float64 of any shape; one K17 launch per call.  `num_bins`, `epsilon` and `adapt` (Keras's approximate
  quantiles) are not offered."""

  def __init__(self, bin_boundaries=None, num_bins=None, epsilon=0.01, output_mode="int", sparse=False, name=None):
    super().__init__()
    if num_bins is not None:
      if bin_boundaries is not None:
        raise ValueError("Both `num_bins` and `bin_boundaries` should not be set.")
      raise NotImplementedError("num_bins (bucket boundaries from adapt) is not supported; pass bin_boundaries")
    if epsilon != 0.01:
      raise NotImplementedError("epsilon only applies to adapt, which is not supported")
    if output_mode != "int":
      if output_mode in _DISCRETIZATION_OUTPUT_MODES:
        raise NotImplementedError(f"output_mode={output_mode!r} is not supported; only 'int' is")
      raise ValueError(f"Unknown output_mode {output_mode!r}; expected one of {('int',) + _DISCRETIZATION_OUTPUT_MODES}")
    if sparse:
      raise NotImplementedError("sparse=True is not supported")
    if bin_boundaries is None:
      raise NotImplementedError("Discretization without bin_boundaries needs adapt, which is not supported")
    b = np.asarray(bin_boundaries, dtype=np.float64)
    if b.ndim != 1:
      raise ValueError(f"bin_boundaries must be a 1-D list, got shape {b.shape}")
    b32 = b.astype(np.float32)
    if np.isnan(b32).any() or (b32[1:] < b32[:-1]).any():
      raise ValueError("bin_boundaries must be sorted (after rounding to float32) and not NaN")
    self.bin_boundaries = b.tolist()
    self._b32 = b32
    self._bounds: Dict[torch.device, torch.Tensor] = {}
    self.output_mode, self.name = output_mode, name

  def adapt(self, data, batch_size=None, steps=None) -> None:
    raise NotImplementedError("Discretization.adapt (approximate quantiles) is not supported; pass bin_boundaries")

  def forward(self, inputs) -> torch.Tensor:
    x = _numeric_input(inputs, "Discretization")
    b = self._bounds.get(x.device)
    if b is None:
      b = self._bounds[x.device] = torch.from_numpy(self._b32).to(x.device)
    return ops.bucketize(x, b)

  def get_config(self) -> Dict[str, Any]:
    return {"name": self.name, "bin_boundaries": list(self.bin_boundaries), "num_bins": None, "epsilon": 0.01,
            "output_mode": self.output_mode, "sparse": False}

  @classmethod
  def from_config(cls, config: Dict[str, Any]):
    return cls(**config)


class Normalization(torch.nn.Module):
  """`tf.keras.layers.Normalization(axis, mean, variance, invert)`: (f32(x) - mean) / max(sqrt(var), 1e-7) as float32, or
  mean + f32(x) * max(sqrt(var), 1e-7) with invert=True.  `axis` is None (one mean and variance) or -1 (one per index
  of the last axis).  The statistics come from `mean` / `variance`, or from `adapt`, which merges batches as Keras's
  update_state does, on the device (K17).  Inputs are CUDA or NumPy int32 / int64 / float32 / float64; the layer
  preprocesses data, so an input that requires grad raises NotImplementedError."""

  def __init__(self, axis=-1, mean=None, variance=None, invert=False, name=None):
    super().__init__()
    if isinstance(axis, (list, tuple)) and len(axis) == 1:
      axis = axis[0]
    if axis is not None and axis != -1:
      raise NotImplementedError(f"axis={axis!r} is not supported; only None and -1 (the last axis) are")
    if (mean is None) != (variance is None):
      raise ValueError("When setting values directly, both `mean` and `variance` must be set. "
                       f"Got mean: {mean} and variance: {variance}")
    self.axis, self.invert, self.name = axis, bool(invert), name
    self.input_mean = None if mean is None else np.asarray(mean, np.float32)
    self.input_variance = None if variance is None else np.asarray(variance, np.float32)
    if axis is None and mean is not None and (self.input_mean.size != 1 or self.input_variance.size != 1):
      raise ValueError("With axis=None, mean and variance must be scalars")
    self._state: Optional[torch.Tensor] = None       # float32 [2, C] on the device: mean, variance
    self._count: Optional[torch.Tensor] = None       # int64 [1]: the values adapt has seen per channel

  def _channels(self, shape) -> int:
    if self.axis is None:
      return 1
    if len(shape) < 2:
      raise NotImplementedError(f"axis=-1 takes inputs of rank >= 2 (one statistic per last index), got shape "
                                f"{tuple(shape)}; reshape to [N, 1] or use axis=None")
    return int(shape[-1])

  def _reset(self, C: int, device) -> None:
    self._state = torch.tensor([[0.0] * C, [1.0] * C], dtype=torch.float32, device=device)
    self._count = torch.zeros((1,), dtype=torch.int64, device=device)

  def adapt(self, data, batch_size=None, steps=None) -> None:
    """Mean and variance from `data`: an array or a tensor, cut into batches of `batch_size` rows (32 by default, as in
    Keras), or a `data.Dataset` whose elements are the batches.  The host reads nothing."""
    if self.input_mean is not None:
      raise ValueError("Cannot adapt a Normalization layer that was given mean and variance")
    if isinstance(data, Dataset):
      rows, parts = None, list(data)
    else:
      rows, parts = int(batch_size or 32), [data]
    self._state = None
    for el in parts:
      C = self._channels(tuple(el.shape) if isinstance(el, torch.Tensor) else np.shape(el) or (1,))
      x = _numeric_input(el, "Normalization.adapt")
      if x.dim() == 0:
        x = x.reshape(1)
      if self._state is None:
        self._reset(C, x.device)
      elif self._state.shape[1] != C:
        raise ValueError(f"Normalization.adapt: a batch with {C} channels after one with {self._state.shape[1]}")
      ops.normalization_adapt(x, C, rows if rows is not None else max(x.shape[0], 1), self._state, self._count)

  @property
  def mean(self) -> Optional[torch.Tensor]:
    return None if self._state is None else self._state[0]

  @property
  def variance(self) -> Optional[torch.Tensor]:
    return None if self._state is None else self._state[1]

  def _statistics(self, shape, device):
    C = self._channels(shape)
    if self.input_mean is not None:
      try:
        m = np.broadcast_to(self.input_mean.reshape(-1) if self.input_mean.size > 1 else self.input_mean.reshape(()), (C,))
        v = np.broadcast_to(self.input_variance.reshape(-1) if self.input_variance.size > 1 else
                            self.input_variance.reshape(()), (C,))
      except ValueError:
        raise ValueError(f"mean / variance of shape {self.input_mean.shape} do not broadcast to {C} channels") from None
      if self._state is None or self._state.device != device or self._state.shape[1] != C:
        self._state = torch.from_numpy(np.stack([m, v]).astype(np.float32)).to(device)
    elif self._state is None:
      self._reset(C, device)
    elif self._state.shape[1] != C:
      raise ValueError(f"Normalization was adapted on {self._state.shape[1]} channels, the input has {C}")
    elif self._state.device != device:
      self._state, self._count = self._state.to(device), self._count.to(device)
    return self._state[0], self._state[1]

  def forward(self, inputs) -> torch.Tensor:
    if isinstance(inputs, torch.Tensor) and inputs.requires_grad:
      raise NotImplementedError("Normalization preprocesses data; an input that requires grad is not supported")
    x = _numeric_input(inputs, "Normalization")
    mean, var = self._statistics(x.shape, x.device)
    return ops.normalize(x, mean, var, self.invert)

  # -- checkpointing and config ---------------------------------------------------------------------------------------
  def get_extra_state(self):
    if self._state is None or self.input_mean is not None:
      return {}
    return {"state": self._state.cpu(), "count": self._count.cpu()}

  def set_extra_state(self, state):
    if state:
      dev = _device()
      self._state, self._count = state["state"].to(dev), state["count"].to(dev)

  def get_config(self) -> Dict[str, Any]:
    return {"name": self.name, "axis": self.axis, "invert": self.invert,
            "mean": None if self.input_mean is None else self.input_mean.tolist(),
            "variance": None if self.input_variance is None else self.input_variance.tolist()}

  @classmethod
  def from_config(cls, config: Dict[str, Any]):
    return cls(**config)


# ---------------------------------------------------------------------------------------------------------------------
# Feature hashing (DESIGN.md §2, A22): Hashing (K18)
# ---------------------------------------------------------------------------------------------------------------------
_HASHING_OUTPUT_MODES = ("one_hot", "multi_hot", "count")


def _is_int(x) -> bool:
  return isinstance(x, (int, np.integer)) and not isinstance(x, (bool, np.bool_))


class Hashing(torch.nn.Module):
  """`tf.keras.layers.Hashing(num_bins, mask_value, salt)` with output_mode="int": each value -> its int64 bin, as
  tf-keras's `_hash_values_to_bins` computes it.  Without a salt the bin is FarmHash Fingerprint64 mod num_bins
  (`tf.strings.to_hash_bucket_fast`); with one it is SipHash-2-4 keyed by the salt (`to_hash_bucket_strong`); an int
  salt s is the key [s, s].  Integers are hashed as their decimal text (`tf.as_string`).  With a `mask_value` and
  num_bins > 1, bin 0 is the mask's and every other value goes to 1 + h mod (num_bins - 1).

  Inputs are CUDA int32 / int64 tensors of any shape (one K18 launch), NumPy or list ints (uploaded once), or NumPy str /
  bytes / object arrays or lists of strings of any shape (`str` encoded as UTF-8, packed on the host and copied to the
  device once, as StringLookup does; trailing NUL bytes are lost the same way).  The output is an int64 CUDA tensor of
  the input's shape.  There is no CPU path: a CPU tensor raises TypeError."""

  def __init__(self, num_bins, mask_value=None, salt=None, output_mode="int", sparse=False, name=None):
    super().__init__()
    if num_bins is None or not _is_int(num_bins) or num_bins <= 0:
      raise ValueError(f"The `num_bins` for `Hashing` cannot be `None` or non-positive values. Received: "
                       f"num_bins={num_bins!r}.")
    if num_bins >= 2**63:
      raise ValueError(f"num_bins must be below 2^63, got {num_bins}")
    if output_mode != "int":
      if output_mode in _HASHING_OUTPUT_MODES:
        raise NotImplementedError(f"output_mode={output_mode!r} is not supported; only 'int' is")
      raise ValueError(f"Unknown output_mode {output_mode!r}; expected one of {('int',) + _HASHING_OUTPUT_MODES}")
    if sparse:
      raise NotImplementedError("sparse=True is not supported")
    if salt is not None:
      if isinstance(salt, (tuple, list)) and len(salt) == 2 and all(_is_int(s) for s in salt):
        salt = [int(s) for s in salt]
      elif _is_int(salt):
        salt = [int(salt), int(salt)]
      else:
        raise ValueError(f"The `salt` argument for `Hashing` can only be a tuple of size 2 integers, or a single "
                         f"integer. Received: salt={salt!r}.")
      if not all(-2**63 <= s < 2**64 for s in salt):
        raise ValueError(f"salt values must fit in 64 bits, got {salt}")
    if mask_value is not None and not (_is_int(mask_value) or isinstance(mask_value, (str, bytes))):
      raise ValueError(f"mask_value must be an int, a str, bytes or None, got {mask_value!r}")
    self.num_bins = int(num_bins)
    self.mask_value = int(mask_value) if _is_int(mask_value) else mask_value
    self.salt = salt
    self.output_mode, self.sparse, self.name = output_mode, False, name

  def _int_mask(self):
    if self.mask_value is not None and not _is_int(self.mask_value):
      raise TypeError(f"Hashing: the string mask_value {self.mask_value!r} cannot mask integer inputs")
    return self.mask_value

  def forward(self, inputs) -> torch.Tensor:
    if isinstance(inputs, tuple) and len(inputs) == 2:
      raise NotImplementedError("ragged (values, row_splits) inputs are not supported")
    if isinstance(inputs, torch.Tensor):
      if not inputs.is_cuda:
        raise TypeError(f"Hashing takes CUDA tensors (there is no CPU path), got one on {inputs.device}")
      if inputs.dtype not in (torch.int32, torch.int64):
        raise TypeError(f"Hashing takes int32 / int64 tensors or strings, got {inputs.dtype}")
      return ops.hashing(inputs, self.num_bins, self.salt, self._int_mask())
    try:
      a = np.asarray(inputs, dtype=object) if isinstance(inputs, (list, tuple)) else np.asarray(inputs)
    except ValueError:
      raise NotImplementedError("ragged inputs are not supported") from None
    if a.dtype.kind == "O":
      a = a.astype(np.int64) if all(_is_int(v) for v in a.flat) else StringLookup._strings(a)
    if a.dtype.kind in "iu":
      if a.dtype.kind == "u" and a.size and a.max() > np.iinfo(np.int64).max:
        raise ValueError("Hashing: unsigned values must fit in int64")
      x = torch.from_numpy(np.ascontiguousarray(a if a.dtype in (np.int32, np.int64) else a.astype(np.int64)))
      return ops.hashing(x.to(_device()), self.num_bins, self.salt, self._int_mask())
    if a.dtype.kind not in "US":
      raise TypeError(f"Hashing takes integers or strings, got dtype {a.dtype}")
    if self.mask_value is not None and _is_int(self.mask_value):
      raise TypeError(f"Hashing: the integer mask_value {self.mask_value} cannot mask string inputs")
    data, offsets, shape = pack_strings(a if a.size else np.zeros(a.shape, "S1"))
    dev = _device()
    if self.mask_value is None:
      byts, offs = upload_packed(data, offsets, dev)
      mask = None
    else:
      byts, offs, mask = upload_packed(data, offsets, dev, np.frombuffer(StringLookup._as_bytes(self.mask_value), np.uint8))
    return ops.hashing((byts, offs), self.num_bins, self.salt, mask).reshape(shape)

  def get_config(self) -> Dict[str, Any]:
    return {"name": self.name, "num_bins": self.num_bins, "mask_value": self.mask_value,
            "salt": None if self.salt is None else list(self.salt), "output_mode": self.output_mode,
            "sparse": self.sparse}

  @classmethod
  def from_config(cls, config: Dict[str, Any]):
    return cls(**config)
