"""Base model: mirror of tensorflow_recommenders/models/base.py (train_step / test_step around a
user-defined `compute_loss`), with a minimal `compile` / `fit` / `evaluate` driver standing in for Keras."""
from __future__ import annotations

from typing import Dict, Iterable, List

import torch

from . import optimizers as _opt
from .backend import learning_phase_scope


class Model(torch.nn.Module):
  """Base model for TFRS models (models/base.py:21-104)."""

  def __init__(self):
    super().__init__()
    self.optimizer = None

  def compute_loss(self, inputs, training: bool = False) -> torch.Tensor:
    raise NotImplementedError("Implementers must implement the `compute_loss` method.")

  # -- Keras-like plumbing -----------------------------------------------------------------------
  def compile(self, optimizer=None) -> None:
    self.optimizer = optimizer if optimizer is not None else _opt.Adagrad(0.001)
    if hasattr(self.optimizer, "bind"):
      self.optimizer.bind(self)

  @property
  def losses(self) -> List[torch.Tensor]:
    """Regularisation losses collected from sublayers (Keras `model.losses`, base.py:71-75)."""
    out = []
    for m in self.modules():
      if m is self:
        continue
      l = getattr(m, "losses", None)
      if isinstance(l, (list, tuple)):
        out.extend(l)
    return out

  @property
  def metrics(self):
    seen, out = set(), []
    for m in self.modules():
      if m is self:
        continue
      ms = getattr(m, "metrics", None)
      if isinstance(ms, (list, tuple)):
        for x in ms:
          if id(x) not in seen:
            seen.add(id(x)); out.append(x)
    return out

  def _regularization_loss(self, like: torch.Tensor) -> torch.Tensor:
    losses = self.losses
    if not losses:
      return torch.zeros((), device=like.device)
    return torch.stack([l.sum() for l in losses]).sum()

  def train_step(self, inputs) -> Dict[str, object]:
    """Custom train step using the `compute_loss` method (base.py:64-85).  `compute_loss` runs in a training learning
    phase (backend.py), so Dropout and BatchNormalization in the towers train without `training` forwarded to them."""
    if self.optimizer is None:
      raise RuntimeError("call compile(optimizer) before train_step")
    self.optimizer.zero_grad()
    with learning_phase_scope(True):
      loss = self.compute_loss(inputs, training=True)
    regularization_loss = self._regularization_loss(loss)
    total_loss = loss + regularization_loss
    total_loss.backward()
    self.optimizer.apply_gradients()
    metrics = {metric.name: metric.result() for metric in self.metrics}
    metrics["loss"] = loss.detach()
    metrics["regularization_loss"] = regularization_loss.detach()
    metrics["total_loss"] = total_loss.detach()
    return metrics

  @torch.no_grad()
  def test_step(self, inputs) -> Dict[str, object]:
    """Custom test step using the `compute_loss` method (base.py:87-104)."""
    with learning_phase_scope(False):
      loss = self.compute_loss(inputs, training=False)
    regularization_loss = self._regularization_loss(loss)
    total_loss = loss + regularization_loss
    metrics = {metric.name: metric.result() for metric in self.metrics}
    metrics["loss"] = loss
    metrics["regularization_loss"] = regularization_loss
    metrics["total_loss"] = total_loss
    return metrics

  def fit(self, data: Iterable, epochs: int = 1) -> List[Dict[str, object]]:
    history = []
    for _ in range(epochs):
      for m in self.metrics:
        m.reset_states()
      last = {}
      for batch in data:
        last = self.train_step(batch)
      history.append(last)
    return history

  def evaluate(self, data: Iterable, return_dict: bool = True):
    for m in self.metrics:
      m.reset_states()
    last = {}
    for batch in data:
      last = self.test_step(batch)
    return last
