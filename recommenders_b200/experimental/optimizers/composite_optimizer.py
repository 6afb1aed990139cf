"""CompositeOptimizer: mirror of tensorflow_recommenders/experimental/optimizers/composite_optimizer.py:25-131.  Routes
disjoint sets of a model's variables to different optimizers, e.g. ClippyAdagrad for the embedding tables and Adagrad for
the dense layers."""
from __future__ import annotations

from typing import Callable, Dict, List, Sequence, Tuple

import torch

from ...layers.embedding import Embedding
from ...optimizers import clear_grads, dense_variables, embedding_tables


class CompositeOptimizer:
  """`CompositeOptimizer([(optimizer, lambda: variables), ...])`.  Each callable returns the variables its optimizer
  updates: `torch.nn.Parameter`s and / or `layers.embedding.Embedding` modules.  A table may also be named by its
  `weight` or by its autograd anchor parameter, so `lambda: list(model.parameters())` and
  `lambda: model.embedding_trainable_variables` both work.  The callables are evaluated again on every step, so layers
  that build their weights on the first forward are picked up."""

  def __init__(self, optimizers_and_vars: Sequence[Tuple[object, Callable[[], Sequence[object]]]],
               name: str = "CompositeOptimizer") -> None:
    if not optimizers_and_vars:
      raise ValueError("`optimizers_and_vars` can't be empty")
    self.name = name
    self._optimizers_and_vars = list(optimizers_and_vars)
    self._module = None

  def bind(self, module: torch.nn.Module) -> "CompositeOptimizer":
    self._module = module
    return self

  def _tables_by_tensor(self) -> Dict[int, Embedding]:
    """id(anchor) and id(weight) -> the table they stand for."""
    out = {}
    if self._module is not None:
      for t in embedding_tables(self._module):
        out[id(t._anchor)] = t
        out[id(t.weight)] = t
    return out

  def _assignment(self) -> List[List[object]]:
    """Each optimizer's variables; ValueError when a variable is claimed twice, or a trainable variable of the bound
    model is claimed by none (composite_optimizer.py:77-97)."""
    tables = self._tables_by_tensor()
    owner: Dict[int, object] = {}
    subsets = []
    for optimizer, var_callable in self._optimizers_and_vars:
      subset = []
      for v in var_callable():
        if isinstance(v, torch.Tensor):
          v = tables.get(id(v), v)
        if id(v) in owner:
          raise ValueError(
              f"The set of variables handled by each optimizer should be "
              f"disjoint, but variable {_describe(v)} is handled both "
              f"by {owner[id(v)]} and {optimizer}.")
        owner[id(v)] = optimizer
        subset.append(v)
      subsets.append(subset)
    if self._module is not None:
      for v in embedding_tables(self._module) + dense_variables(self._module):
        if id(v) not in owner:
          raise ValueError(f"Variable {_describe(v)} is not handled by any optimizer. "
                           f"This would cause it to be not trained.")
    return subsets

  def apply_gradients(self) -> None:
    """Hands each optimizer its own variables (composite_optimizer.py:73-105).  Every check runs before any update."""
    subsets = self._assignment()
    for (optimizer, _), subset in zip(self._optimizers_and_vars, subsets):
      optimizer.apply_gradients(subset)

  step = apply_gradients

  def zero_grad(self) -> None:
    if self._module is not None:
      clear_grads(embedding_tables(self._module), dense_variables(self._module))
    for optimizer, _ in self._optimizers_and_vars:
      optimizer.zero_grad()

  def get_config(self):
    raise NotImplementedError("CompositeOptimizer cannot be serialized because"
                              " it uses callable to get variables.")

  @property
  def iterations(self) -> int:
    """The first optimizer's step count (composite_optimizer.py:107-111)."""
    return self._optimizers_and_vars[0][0].iterations

  def variables(self) -> List[torch.Tensor]:
    """The state of every optimizer, in the order of the optimizers."""
    out = []
    for optimizer, _ in self._optimizers_and_vars:
      out += optimizer.variables()
    return out

  @property
  def optimizers(self) -> List[object]:
    """The optimizers, in the original order."""
    return [optimizer for optimizer, _ in self._optimizers_and_vars]


def _describe(v) -> str:
  if isinstance(v, Embedding):
    return f"Embedding({v.input_dim}, {v.output_dim})"
  return f"Parameter(shape={tuple(v.shape)})"
