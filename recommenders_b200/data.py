"""A minimal stand-in for the slice of `tf.data.Dataset` the reference's retrieval path uses
(`from_tensor_slices`, `batch`, `zip`, `map`, iteration) so candidate corpora can be written the same
way as in the reference (`tf.data.Dataset.from_tensor_slices(c).batch(128)`, README.md:71).
Elements are CUDA torch tensors (embeddings / integer ids) or NumPy arrays (e.g. string identifiers), or tuples or dicts of
them."""
from __future__ import annotations

from typing import Callable, Iterable, Iterator, List, Sequence, Tuple, Union

import numpy as np
import torch

Element = Union[torch.Tensor, np.ndarray, Tuple, dict]


def _slice(x, lo, hi):
  if isinstance(x, tuple):
    return tuple(_slice(e, lo, hi) for e in x)
  if isinstance(x, dict):
    return {k: _slice(v, lo, hi) for k, v in x.items()}
  return x[lo:hi]


def _len(x) -> int:
  if isinstance(x, tuple):
    return _len(x[0])
  if isinstance(x, dict):
    return _len(next(iter(x.values())))
  return int(x.shape[0])


class Dataset:
  """Re-iterable sequence of batches."""

  def __init__(self, factory: Callable[[], Iterator[Element]], is_tuple: bool):
    self._factory = factory
    self.is_tuple = is_tuple

  def __iter__(self) -> Iterator[Element]:
    return self._factory()

  @staticmethod
  def from_tensor_slices(tensors) -> "Dataset":
    if isinstance(tensors, dict):
      tensors = {k: v if isinstance(v, (torch.Tensor, np.ndarray)) else np.asarray(v) for k, v in tensors.items()}
      if not tensors:
        raise ValueError("from_tensor_slices needs at least one feature")
      n = _len(tensors)
      if any(_len(v) != n for v in tensors.values()):
        raise ValueError(f"All features have to have the same batch dimension. Got { {k: _len(v) for k, v in tensors.items()} }.")
      return _Slices(tensors)
    if isinstance(tensors, list):
      tensors = tuple(tensors)
    if isinstance(tensors, tuple):
      n = _len(tensors)
      if any(_len(t) != n for t in tensors):
        raise ValueError("Candidates and identifiers have to have the same batch dimension. "
                         f"Got {[_len(t) for t in tensors]}.")
    return _Slices(tensors)

  @staticmethod
  def from_batches(batches: Sequence[Element]) -> "Dataset":
    batches = list(batches)
    return Dataset(lambda: iter(batches), bool(batches) and isinstance(batches[0], tuple))

  @staticmethod
  def zip(datasets: Tuple["Dataset", ...]) -> "Dataset":
    datasets = tuple(datasets)

    def gen():
      for els in zip(*datasets):
        yield tuple(els)
    return Dataset(gen, True)

  def batch(self, batch_size: int, drop_remainder: bool = False) -> "Dataset":
    raise NotImplementedError("batch() is only defined on from_tensor_slices datasets")

  def map(self, fn: Callable) -> "Dataset":
    src = self

    def gen():
      for el in src:
        yield fn(*el) if isinstance(el, tuple) else fn(el)
    return Dataset(gen, self.is_tuple)


class _Slices(Dataset):

  def __init__(self, tensors):
    self._tensors = tensors
    super().__init__(lambda: iter([tensors]), isinstance(tensors, tuple))

  def batch(self, batch_size: int, drop_remainder: bool = False) -> Dataset:
    t = self._tensors
    n = _len(t)

    def gen():
      for lo in range(0, n, batch_size):
        hi = min(lo + batch_size, n)
        if drop_remainder and hi - lo < batch_size:
          return
        yield _slice(t, lo, hi)
    return Dataset(gen, isinstance(t, tuple))


def as_dataset(obj) -> Dataset:
  if isinstance(obj, Dataset):
    return obj
  if isinstance(obj, (list, tuple)):
    return Dataset.from_batches(obj)
  if hasattr(obj, "__iter__"):
    return Dataset.from_batches(list(obj))
  raise TypeError(f"cannot interpret {type(obj)} as a dataset of candidate batches")
