"""Adagrad with the sparse row update of the retrieval hot path (the optimizer the reference's README
passes to `model.compile`, README.md:84: `tf.keras.optimizers.Adagrad(0.5)`).

Keras defaults: initial_accumulator_value=0.1, epsilon=1e-7.  `eps_inside_sqrt=True` is the Keras-3 /
tf-keras `optimizers.Adagrad` rule  var -= lr*g/sqrt(acc+eps); False is the legacy
`optimizers.legacy.Adagrad` rule  var -= lr*g/(sqrt(acc)+eps)  (SURVEY.md A10 -- third-party, unpinned).

Adam: tf-keras's legacy `optimizers.legacy.Adam` rules on the K10 kernels (DESIGN.md A15).
Ftrl: tf-keras's legacy `optimizers.legacy.Ftrl` rules on the K12 kernels (DESIGN.md A17)."""
from __future__ import annotations

from typing import Any, Dict, Iterable, List, Optional, Sequence, Tuple, Union

import torch

from . import ops
from .layers.embedding import Embedding

Variable = Union[Embedding, torch.nn.Parameter]


def embedding_tables(module: torch.nn.Module) -> List[Embedding]:
  """The embedding tables of a model (updated from their sparse (ids, rows) gradients)."""
  return [m for m in module.modules() if isinstance(m, Embedding)]


def dense_variables(module: torch.nn.Module) -> List[torch.nn.Parameter]:
  """The trainable parameters of a model other than the tables' autograd anchors."""
  anchors = {id(t._anchor) for t in embedding_tables(module)}
  return [p for p in module.parameters() if p.requires_grad and id(p) not in anchors]


def split_variables(variables: Iterable[Variable]) -> Tuple[List[Embedding], List[torch.nn.Parameter]]:
  tables, dense = [], []
  for v in variables:
    if isinstance(v, Embedding):
      tables.append(v)
    elif isinstance(v, torch.Tensor):
      dense.append(v)
    else:
      raise TypeError(f"cannot optimize a {type(v).__name__}: expected an Embedding or a torch.nn.Parameter")
  return tables, dense


def clear_grads(tables: Sequence[Embedding], dense: Sequence[torch.Tensor]) -> None:
  for p in dense:
    p.grad = None
  for t in tables:
    t.pop_sparse_grads()
    t._anchor.grad = None


class _SlotOptimizer:
  """Variable discovery and per-variable slots shared by Adagrad, ClippyAdagrad, Adam, Ftrl and SGD."""

  def __init__(self):
    self.iterations = 0
    self._module = None
    self._dense: List[torch.nn.Parameter] = []
    self._tables: List[Embedding] = []
    self._slots = {}

  def bind(self, module: torch.nn.Module):
    """Attach to a model.  The variable lists are re-read on every step (`_refresh`), like the reference's
    `self.trainable_variables` at models/base.py:77: layers that create their weights lazily on the first
    forward (Cross, MultiLayerDCN) are picked up even when compile() ran before the first batch."""
    self._module = module
    self._refresh()
    return self

  def _refresh(self) -> None:
    if self._module is None:
      return
    self._tables = embedding_tables(self._module)
    self._dense = dense_variables(self._module)

  def _slot(self, owner, attr: str, like: torch.Tensor, value: float) -> torch.Tensor:
    """The slot `attr` of a variable, filled with `value` when created, stored ON its owner object (an Embedding module
    or a Parameter) so it lives and dies with it -- an id()-keyed dict would hand a recycled id the previous owner's
    state."""
    a = getattr(owner, attr, None)
    if a is None or a.shape != like.shape or a.device != like.device:
      a = torch.full_like(like, value)
      setattr(owner, attr, a)
      self._slots[(id(owner), attr)] = a
    return a

  @staticmethod
  def _table_grads(t: Embedding) -> Optional[Tuple[torch.Tensor, torch.Tensor]]:
    """A table's gradient for this step, taken off the table: the (ids, rows) of all its lookups concatenated, one
    variable like the IndexedSlices of the reference; None when no lookup has one."""
    grads = t.pop_sparse_grads()
    if not grads:
      return None
    return torch.cat([i.reshape(-1) for i, _ in grads], 0), torch.cat([g.reshape(-1, t.output_dim) for _, g in grads], 0)

  def zero_grad(self):
    self._refresh()
    clear_grads(self._tables, self._dense)

  @torch.no_grad()
  def apply_gradients(self, variables: Optional[Iterable[Variable]] = None):
    """optimizer.apply_gradients(zip(grads, vars)) -- models/base.py:78.  Updates the bound model's variables, or only
    `variables` (Embedding modules and Parameters) when given."""
    if variables is None:
      self._refresh()
      tables, dense = self._tables, self._dense
    else:
      tables, dense = split_variables(variables)
    self._apply(tables, dense)
    self.iterations += 1

  def step(self, variables: Optional[Iterable[Variable]] = None):
    return self.apply_gradients(variables)

  def _apply(self, tables: Sequence[Embedding], dense: Sequence[torch.nn.Parameter]) -> None:
    raise NotImplementedError

  def variables(self) -> List[torch.Tensor]:
    """The optimizer's state: its slots of every variable it has updated."""
    return list(self._slots.values())


class _AccumulatorOptimizer(_SlotOptimizer):
  """One accumulator slot per variable (Adagrad and ClippyAdagrad)."""

  _ACC_ATTR = "_tfrs_adagrad_acc"

  def __init__(self, initial_accumulator_value: float):
    super().__init__()
    self.initial_accumulator_value = initial_accumulator_value

  def _accum(self, owner, like: torch.Tensor) -> torch.Tensor:
    return self._slot(owner, self._ACC_ATTR, like, self.initial_accumulator_value)

  def state_dict(self):
    return {"acc": {k: v.clone() for (k, _), v in self._slots.items()}}


class Adagrad(_AccumulatorOptimizer):

  def __init__(self, learning_rate: float = 0.001, initial_accumulator_value: float = 0.1, epsilon: float = 1e-7,
               eps_inside_sqrt: bool = True):
    super().__init__(initial_accumulator_value)
    self.learning_rate = learning_rate
    self.epsilon = epsilon
    self.eps_inside_sqrt = eps_inside_sqrt

  def _apply(self, tables, dense):
    for t in tables:
      g = self._table_grads(t)
      if g is not None:
        ops.sparse_adagrad_(t.weight, self._accum(t, t.weight), *g, self.learning_rate, self.epsilon, self.eps_inside_sqrt)
    for p in dense:
      if p.grad is None:
        continue
      a = self._accum(p, p)
      g = p.grad
      a.addcmul_(g, g)
      den = (a + self.epsilon).sqrt_() if self.eps_inside_sqrt else a.sqrt().add_(self.epsilon)
      p.addcdiv_(g, den, value=-self.learning_rate)


class Adam(_SlotOptimizer):
  """Adam with tf-keras's legacy rules (`tf.keras.optimizers.legacy.Adam`, optimizer_v2/adam.py; DESIGN.md section 2).
  Dense variables take the dense rule.  An embedding table takes the sparse rule: every step decays `m` and `v` over
  the whole table and moves every row whose `m` is nonzero, touched or not, like tf-keras's `_resource_apply_sparse` on
  CPU / GPU.  With `lazy_embeddings=True` only the rows of the step's ids are updated and the other rows keep their
  variable, `m` and `v` bit for bit, as TPU embedding engines do by default; for a large table that is the cheap choice.

  The slots `m` and `v` start at zero.  `amsgrad=True` raises NotImplementedError."""

  _M_ATTR = "_tfrs_adam_m"
  _V_ATTR = "_tfrs_adam_v"

  def __init__(self, learning_rate: float = 0.001, beta_1: float = 0.9, beta_2: float = 0.999, epsilon: float = 1e-7,
               amsgrad: bool = False, lazy_embeddings: bool = False, name: str = "Adam"):
    if amsgrad:
      raise NotImplementedError("Adam: amsgrad=True is not supported")
    super().__init__()
    self.learning_rate = learning_rate
    self.beta_1 = beta_1
    self.beta_2 = beta_2
    self.epsilon = epsilon
    self.amsgrad = amsgrad
    self.lazy_embeddings = lazy_embeddings
    self.name = name

  def _apply(self, tables, dense):
    alpha = ops.adam_alpha(self.learning_rate, self.beta_1, self.beta_2, self.iterations + 1)
    rule = dict(alpha=alpha, beta_1=self.beta_1, beta_2=self.beta_2, epsilon=self.epsilon)
    for t in tables:
      g = self._table_grads(t)
      if g is not None:
        ops.sparse_adam_(t.weight, self._slot(t, self._M_ATTR, t.weight, 0.0), self._slot(t, self._V_ATTR, t.weight, 0.0),
                         *g, lazy=self.lazy_embeddings, **rule)
    params = [p for p in dense if p.grad is not None]
    if params:
      ops.adam_dense_(params, [p.grad for p in params], [self._slot(p, self._M_ATTR, p, 0.0) for p in params],
                      [self._slot(p, self._V_ATTR, p, 0.0) for p in params], **rule)

  def get_config(self) -> Dict[str, Any]:
    return {"name": self.name, "learning_rate": self.learning_rate, "beta_1": self.beta_1, "beta_2": self.beta_2,
            "epsilon": self.epsilon, "amsgrad": self.amsgrad, "lazy_embeddings": self.lazy_embeddings}

  @classmethod
  def from_config(cls, config: Dict[str, Any]) -> "Adam":
    return cls(**config)


class Ftrl(_SlotOptimizer):
  """FTRL-Proximal with tf-keras's legacy rules (`tf.keras.optimizers.legacy.Ftrl`, optimizer_v2/ftrl.py; DESIGN.md
  section 2).  Dense variables and embedding tables take the same element rule; a table updates only the rows of the
  step's ids (duplicates summed), and every other row keeps its variable, accumulator and linear slot bit for bit, as
  tf-keras's `_resource_apply_sparse` does.  `beta` is folded into the l2 strength once per step (`ops.ftrl_l2`).

  The accumulator starts at `initial_accumulator_value`, the linear slot at zero."""

  _ACC_ATTR = "_tfrs_ftrl_acc"
  _LIN_ATTR = "_tfrs_ftrl_linear"

  def __init__(self, learning_rate: float = 0.001, learning_rate_power: float = -0.5,
               initial_accumulator_value: float = 0.1, l1_regularization_strength: float = 0.0,
               l2_regularization_strength: float = 0.0, name: str = "Ftrl",
               l2_shrinkage_regularization_strength: float = 0.0, beta: float = 0.0):
    if initial_accumulator_value < 0.0:
      raise ValueError(f"`initial_accumulator_value` needs to be positive or zero, received: {initial_accumulator_value}")
    if learning_rate_power > 0.0:
      raise ValueError(f"`learning_rate_power` needs to be negative or zero, received: {learning_rate_power}")
    for arg, value in (("l1_regularization_strength", l1_regularization_strength),
                       ("l2_regularization_strength", l2_regularization_strength),
                       ("l2_shrinkage_regularization_strength", l2_shrinkage_regularization_strength)):
      if value < 0.0:
        raise ValueError(f"`{arg}` needs to be positive or zero, received: {value}")
    super().__init__()
    self.learning_rate = learning_rate
    self.learning_rate_power = learning_rate_power
    self.initial_accumulator_value = initial_accumulator_value
    self.l1_regularization_strength = l1_regularization_strength
    self.l2_regularization_strength = l2_regularization_strength
    self.name = name
    self.l2_shrinkage_regularization_strength = l2_shrinkage_regularization_strength
    self.beta = beta

  def _slots_of(self, owner, like: torch.Tensor):
    return (self._slot(owner, self._ACC_ATTR, like, self.initial_accumulator_value),
            self._slot(owner, self._LIN_ATTR, like, 0.0))

  def _apply(self, tables, dense):
    rule = dict(lr=self.learning_rate, lr_power=self.learning_rate_power, l1=self.l1_regularization_strength,
                l2a=ops.ftrl_l2(self.l2_regularization_strength, self.beta, self.learning_rate),
                l2_shrinkage=self.l2_shrinkage_regularization_strength)
    for t in tables:
      g = self._table_grads(t)
      if g is not None:
        ops.sparse_ftrl_(t.weight, *self._slots_of(t, t.weight), *g, **rule)
    params = [p for p in dense if p.grad is not None]
    if params:
      slots = [self._slots_of(p, p) for p in params]
      ops.ftrl_dense_([p.data for p in params], [p.grad for p in params], [a for a, _ in slots], [z for _, z in slots],
                      **rule)

  def get_config(self) -> Dict[str, Any]:
    return {"name": self.name, "learning_rate": self.learning_rate, "learning_rate_power": self.learning_rate_power,
            "initial_accumulator_value": self.initial_accumulator_value,
            "l1_regularization_strength": self.l1_regularization_strength,
            "l2_regularization_strength": self.l2_regularization_strength,
            "l2_shrinkage_regularization_strength": self.l2_shrinkage_regularization_strength, "beta": self.beta}

  @classmethod
  def from_config(cls, config: Dict[str, Any]) -> "Ftrl":
    return cls(**config)


class SGD(_SlotOptimizer):
  """Plain SGD with tf-keras's legacy rules (`tf.keras.optimizers.legacy.SGD`, optimizer_v2/gradient_descent.py):
  var -= lr * g.  An embedding table applies every occurrence of an id on its own, in order of occurrence, like the
  reference's `resource_scatter_add` without deduplication (the order is unpinned against TF).  Dense variables take one
  multi-tensor launch.  `momentum != 0` and `nesterov=True` raise NotImplementedError."""

  def __init__(self, learning_rate: float = 0.01, momentum: float = 0.0, nesterov: bool = False, name: str = "SGD"):
    if momentum != 0.0 or nesterov:
      raise NotImplementedError("SGD: momentum and nesterov are not supported")
    super().__init__()
    self.learning_rate = learning_rate
    self.momentum = momentum
    self.nesterov = nesterov
    self.name = name

  def _apply(self, tables, dense):
    for t in tables:
      g = self._table_grads(t)
      if g is not None:
        ops.sparse_sgd_(t.weight, *g, self.learning_rate)
    params = [p for p in dense if p.grad is not None]
    if params:
      with torch.no_grad():
        ops.sgd_dense_([p.data for p in params], [p.grad for p in params], self.learning_rate)

  def get_config(self) -> Dict[str, Any]:
    return {"name": self.name, "learning_rate": self.learning_rate, "momentum": self.momentum, "nesterov": self.nesterov}

  @classmethod
  def from_config(cls, config: Dict[str, Any]) -> "SGD":
    return cls(**config)
