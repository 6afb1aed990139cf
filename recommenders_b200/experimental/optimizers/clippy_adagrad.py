"""ClippyAdagrad: mirror of tensorflow_recommenders/experimental/optimizers/clippy_adagrad.py:21-269 (Adagrad with adaptive
clipping, arXiv 2302.09178), on libtfrs_b200's K7 kernels: one sparse call per embedding table and one multi-tensor call
for all dense variables of a step."""
from __future__ import annotations

from typing import Any, Dict, List, Sequence, Tuple, Union

import torch

from ... import ops
from ...layers.embedding import Embedding
from ...optimizers import _AccumulatorOptimizer


def _on_cuda(x, name: str) -> torch.Tensor:
  if isinstance(x, torch.Tensor):
    return ops.require_cuda(x, name)
  return torch.tensor(x, dtype=torch.float32, device=torch.device("cuda", torch.cuda.current_device()))


def shrink_by_references(tensor: Union[torch.Tensor, float], references: Sequence[Union[torch.Tensor, float]],
                         relative_factors: Sequence[float], absolute_factor: float) -> Tuple[torch.Tensor, torch.Tensor]:
  """Scales `tensor` so that |tensor_i| * scale <= sum_j |reference_j,i| * relative_factor_j + absolute_factor for every i,
  with the largest scale in [0, 1] (clippy_adagrad.py:21-70).  Returns (tensor * scale, scale).  Tensors must live on
  a CUDA device; Python numbers are placed on the current one."""
  if any(relative_factor < 0 for relative_factor in relative_factors):
    raise ValueError("relative_factors must all be non-negative.")
  if absolute_factor < 0:
    raise ValueError("absolute_factor must be non-negative.")
  if len(references) != len(relative_factors):
    raise ValueError(
        "references and relative_factors must have the same length. "
        f"Instead they are {len(references)} and {len(relative_factors)}.")
  t = _on_cuda(tensor, "tensor")
  max_delta = torch.full((), float(absolute_factor), dtype=t.dtype, device=t.device)
  for i, (reference, relative_factor) in enumerate(zip(references, relative_factors)):
    max_delta = max_delta + _on_cuda(reference, f"references[{i}]").abs() * relative_factor
  # where(tensor == 0, 1, divide_no_nan(max_delta, |tensor|)): the division only counts where tensor != 0
  abs_t = t.abs()
  per_element_scale = torch.where(abs_t == 0, torch.ones_like(abs_t), max_delta / abs_t)
  scale = torch.clamp(per_element_scale.min(), max=1.0)
  return t * scale, scale


class ClippyAdagrad(_AccumulatorOptimizer):
  """An Adagrad variant with adaptive clipping (clippy_adagrad.py:74-92).  Each variable's step is multiplied by the
  largest factor in [0, 1] that keeps every touched element's change under
    |w| * variable_relative_threshold + accumulator_relative_threshold / sqrt(accum) + absolute_threshold.

  Attributes:
    iterations: the number of steps this optimizer has run.
    clipping_factors: with `export_clipping_factors=True`, one 0-d float32 device tensor per variable (embedding tables,
      then dense variables, in the order they were bound or last given), holding the factor of the last step that
      updated it (0 before that); an empty list otherwise.  Reading it does not synchronise with the device.
  """

  _ACC_ATTR = "_tfrs_clippy_acc"
  _FACTOR_ATTR = "_tfrs_clippy_factor"

  def __init__(self, learning_rate: float = 0.001, initial_accumulator_value: float = 0.1,
               variable_relative_threshold: float = 0.1, accumulator_relative_threshold: float = 0.0,
               absolute_threshold: float = 1e-7, epsilon: float = 1e-7, export_clipping_factors: bool = False,
               clip_accumulator_update: bool = False, use_standard_accumulator_update: bool = False,
               name: str = "ClippyAdagrad") -> None:
    if clip_accumulator_update and use_standard_accumulator_update:
      raise ValueError(
          "clip_accumulator_update and use_standard_accumulator_update cannot "
          "both be set to True.")
    super().__init__(initial_accumulator_value)
    self.name = name
    self.learning_rate = float(learning_rate)
    self.variable_relative_threshold = variable_relative_threshold
    self.accumulator_relative_threshold = accumulator_relative_threshold
    self.absolute_threshold = absolute_threshold
    self.epsilon = epsilon
    self.export_clipping_factors = export_clipping_factors
    self.clip_accumulator_update = clip_accumulator_update
    self.use_standard_accumulator_update = use_standard_accumulator_update
    self._order: List[Any] = []
    self._dense_factors = None   # (variables, [n] buffer, 0-d views) of the last multi-tensor call

  def _refresh(self) -> None:
    super()._refresh()
    if self._module is not None:
      self._order = self._tables + self._dense

  def _rule(self) -> Dict[str, Any]:
    return dict(lr=self.learning_rate, eps=self.epsilon, variable_relative_threshold=self.variable_relative_threshold,
                accumulator_relative_threshold=self.accumulator_relative_threshold,
                absolute_threshold=self.absolute_threshold, clip_accumulator_update=self.clip_accumulator_update,
                use_standard_accumulator_update=self.use_standard_accumulator_update)

  def _factor(self, owner, device) -> torch.Tensor:
    f = getattr(owner, self._FACTOR_ATTR, None)
    if f is None or f.device != device:
      f = torch.zeros((), dtype=torch.float32, device=device)
      setattr(owner, self._FACTOR_ATTR, f)
    return f

  def _dense_factor_buffer(self, params: Sequence[torch.nn.Parameter]) -> torch.Tensor:
    """One [n] buffer for the multi-tensor call; each parameter's factor is a 0-d view of it.  Reused while the set of
    parameters stays the same, so the tensors in `clipping_factors` keep receiving the new factors."""
    cached = self._dense_factors
    if cached is not None and len(cached[0]) == len(params) and all(
        a is b and getattr(b, self._FACTOR_ATTR, None) is view for a, b, view in zip(cached[0], params, cached[2])):
      return cached[1]
    buf = torch.zeros((len(params),), dtype=torch.float32, device=params[0].device)
    views = [buf[i] for i in range(len(params))]
    for p, view in zip(params, views):
      setattr(p, self._FACTOR_ATTR, view)
    self._dense_factors = (list(params), buf, views)
    return buf

  def _apply(self, tables, dense):
    self._order = list(tables) + list(dense)
    rule = self._rule()
    for t in tables:
      g = self._table_grads(t)
      if g is not None:
        factor = self._factor(t, t.weight.device) if self.export_clipping_factors else None
        ops.sparse_clippy_adagrad_(t.weight, self._accum(t, t.weight), *g, clipping_factor=factor, **rule)
    params = [p for p in dense if p.grad is not None]
    if params:
      factors = self._dense_factor_buffer(params) if self.export_clipping_factors else None
      ops.clippy_adagrad_dense_(params, [p.grad for p in params], [self._accum(p, p) for p in params],
                                clipping_factors=factors, **rule)

  @property
  def clipping_factors(self) -> List[torch.Tensor]:
    if not self.export_clipping_factors:
      return []
    return [self._factor(v, v.weight.device if isinstance(v, Embedding) else v.device) for v in self._order]

  def get_config(self) -> Dict[str, Any]:
    """Every constructor argument.  (The reference's get_config, clippy_adagrad.py:256-269, omits
    use_standard_accumulator_update; it is kept here so that from_config restores the same optimizer.)"""
    return {"name": self.name, "learning_rate": self.learning_rate,
            "initial_accumulator_value": self.initial_accumulator_value,
            "variable_relative_threshold": self.variable_relative_threshold,
            "accumulator_relative_threshold": self.accumulator_relative_threshold,
            "absolute_threshold": self.absolute_threshold, "epsilon": self.epsilon,
            "export_clipping_factors": self.export_clipping_factors,
            "clip_accumulator_update": self.clip_accumulator_update,
            "use_standard_accumulator_update": self.use_standard_accumulator_update}

  @classmethod
  def from_config(cls, config: Dict[str, Any]) -> "ClippyAdagrad":
    return cls(**config)
