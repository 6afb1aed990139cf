"""The learning phase: whether a layer whose output depends on `training` (Dropout, BatchNormalization) runs in training
mode.  One rule, `resolve_training`, serves every such layer:

  1. the explicit `training=` argument of the call;
  2. the innermost `learning_phase_scope`;
  3. False.

`Model.train_step` runs `compute_loss` inside `learning_phase_scope(True)` and `test_step` inside
`learning_phase_scope(False)`, so the towers of a model see the phase without forwarding `training` themselves (a
`torch.nn.Sequential` tower cannot take the keyword).  torch's `Module.training` is not consulted: it defaults to True,
which would turn dropout on in a plain call.  DESIGN.md (the training phase) records the difference from tf-keras."""
from __future__ import annotations

import contextlib
import threading
from typing import Iterator, Optional

_state = threading.local()


def _stack() -> list:
  s = getattr(_state, "phases", None)
  if s is None:
    s = _state.phases = []
  return s


@contextlib.contextmanager
def learning_phase_scope(value: bool) -> Iterator[None]:
  """Within the block, a call without an explicit `training=` runs in training mode iff `value`.  Scopes nest; the
  innermost wins.  Per thread."""
  s = _stack()
  s.append(bool(value))
  try:
    yield
  finally:
    s.pop()


def learning_phase() -> Optional[bool]:
  """The innermost scope's phase, or None outside every scope."""
  s = _stack()
  return s[-1] if s else None


def resolve_training(training=None) -> bool:
  """The training flag of a call: `training` when given, else the innermost scope's, else False."""
  if training is not None:
    return bool(training)
  phase = learning_phase()
  return bool(phase) if phase is not None else False
