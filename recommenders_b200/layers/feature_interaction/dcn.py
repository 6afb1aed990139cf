"""Cross layer of DCN-v2: mirror of tensorflow_recommenders/layers/feature_interaction/dcn.py."""
from __future__ import annotations

import math
from typing import Callable, Optional, Union

import torch

from ... import ops

_ACTIVATIONS = {
    None: None, "linear": None,
    "relu": torch.relu, "sigmoid": torch.sigmoid, "tanh": torch.tanh,
    "swish": torch.nn.functional.silu, "silu": torch.nn.functional.silu, "gelu": torch.nn.functional.gelu,
}


def _init(name, shape, device):
  """Keras initializers by name: "truncated_normal" (mean 0, stddev 0.05, cut at 2 sigma), "zeros", "ones",
  "glorot_uniform", "orthogonal" (gain 1); a callable(shape, device) is used as is."""
  if callable(name):
    return name(shape, device)
  if name == "orthogonal":
    # Keras's Orthogonal: q of the QR of a normal (max(rows, cols), min(rows, cols)) matrix, columns scaled by
    # sign(diag(r)), transposed when rows < cols -- orthonormal rows or columns, whichever are fewer.  rows = the product
    # of all dimensions but the last.  Drawn and factorised in float64 on the host from torch's seeded generator.
    rows, cols = math.prod(shape[:-1]), shape[-1]
    q, r = torch.linalg.qr(torch.randn((max(rows, cols), min(rows, cols)), dtype=torch.float64))
    q = q * torch.sign(torch.diagonal(r))
    q = q.T if rows < cols else q
    return q.reshape(shape).to(device=device, dtype=torch.float32).contiguous()
  t = torch.empty(shape, dtype=torch.float32, device=device)
  if name == "truncated_normal":
    torch.nn.init.trunc_normal_(t, mean=0.0, std=0.05, a=-0.1, b=0.1)
  elif name == "zeros":
    t.zero_()
  elif name == "ones":
    t.fill_(1.0)
  elif name == "glorot_uniform":
    torch.nn.init.xavier_uniform_(t)
  else:
    raise ValueError(f"Unknown initializer: {name}")
  return t


class Cross(torch.nn.Module):
  """Cross Layer in Deep & Cross Network (dcn.py:22-208).

  x_{i+1} = x0 .* (W * xi + bias + diag_scale * xi) + xi, W full-rank or low-rank U*V.
  The full-rank, no-preactivation case (the DCN-v2 ranking hot path) is one fused kernel
  (GEMM + bias + diag + x0-multiply + residual); low-rank / preactivation variants compose the exact
  SGEMM with elementwise ops.  `kernel` is stored [in, out] like Keras' Dense (dcn.py:121-130)."""

  def __init__(self, projection_dim: Optional[int] = None, diag_scale: Optional[float] = 0.0, use_bias: bool = True,
               preactivation: Optional[Union[str, Callable]] = None,
               kernel_initializer="truncated_normal", bias_initializer="zeros",
               kernel_regularizer=None, bias_regularizer=None, **kwargs):
    super().__init__()
    self._projection_dim = projection_dim
    self._diag_scale = diag_scale
    self._use_bias = use_bias
    self._preactivation_cfg = preactivation
    self._preactivation = _ACTIVATIONS[preactivation] if (preactivation is None or isinstance(preactivation, str)) else preactivation
    self._kernel_initializer = kernel_initializer
    self._bias_initializer = bias_initializer
    self._kernel_regularizer = kernel_regularizer
    self._bias_regularizer = bias_regularizer
    self._input_dim = None
    self.built = False
    self.name = kwargs.get("name")
    if self._diag_scale < 0:
      raise ValueError("`diag_scale` should be non-negative. Got `diag_scale` = {}".format(self._diag_scale))

  def build(self, input_shape, device=None):
    last_dim = int(input_shape[-1])
    device = device or torch.device("cuda", torch.cuda.current_device())
    self._input_dim = last_dim
    if self._projection_dim is None:
      self.kernel = torch.nn.Parameter(_init(self._kernel_initializer, (last_dim, last_dim), device))
    else:
      self.kernel_u = torch.nn.Parameter(_init(self._kernel_initializer, (last_dim, self._projection_dim), device))
      self.kernel_v = torch.nn.Parameter(_init(self._kernel_initializer, (self._projection_dim, last_dim), device))
    if self._use_bias:
      self.bias = torch.nn.Parameter(_init(self._bias_initializer, (last_dim,), device))
    else:
      self.bias = None
    self.built = True

  @property
  def losses(self):
    """Regularisation terms (Keras collects them in `model.losses`, models/base.py:71-75)."""
    out = []
    if self.built and self._kernel_regularizer is not None:
      ks = [self.kernel] if self._projection_dim is None else [self.kernel_u, self.kernel_v]
      out += [self._kernel_regularizer(k) for k in ks]
    if self.built and self._bias_regularizer is not None and self.bias is not None:
      out.append(self._bias_regularizer(self.bias))
    return out

  def call(self, x0: torch.Tensor, x: Optional[torch.Tensor] = None) -> torch.Tensor:
    if not self.built:
      self.build(x0.shape, x0.device if isinstance(x0, torch.Tensor) else None)
    if x is None:
      x = x0
    if x0.shape[-1] != x.shape[-1]:
      raise ValueError("`x0` and `x` dimension mismatch! Got `x0` dimension {}, and x "
                       "dimension {}. This case is not supported yet.".format(x0.shape[-1], x.shape[-1]))
    lead = x0.shape[:-1]
    # 2-D inputs are passed through as the SAME tensor objects: a stacked layer recognises its predecessor's output (and
    # the statistics its kernel attached to it) by identity
    x0f = x0 if x0.dim() == 2 else x0.reshape(-1, x0.shape[-1])
    xf = x if x.dim() == 2 else x.reshape(-1, x.shape[-1])
    if self._projection_dim is None and self._preactivation is None:
      out = ops.cross(x0f, xf, self.kernel, self.bias, float(self._diag_scale or 0.0))
      return out if len(lead) == 1 else out.reshape(*lead, -1)
    if (self._projection_dim is not None and self._preactivation is None and
        ops.cross_lowrank_supported(xf.shape[0], xf.shape[1], self._projection_dim)):
      # low-rank: two tensor-core GEMMs, the cross formula fused into the second one
      out = ops.cross_lowrank(x0f, xf, self.kernel_u, self.kernel_v, self.bias, float(self._diag_scale or 0.0))
      return out.reshape(*lead, -1)
    if self._projection_dim is None:
      prod = ops.matmul(xf, self.kernel)
    else:
      prod = ops.matmul(ops.matmul(xf, self.kernel_u), self.kernel_v)
    if self.bias is not None:
      prod = prod + self.bias
    if self._preactivation is not None:
      prod = self._preactivation(prod)
    if self._diag_scale:
      prod = prod + self._diag_scale * xf
    return (x0f * prod + xf).reshape(*lead, -1)

  def forward(self, x0, x=None):
    return self.call(x0, x)

  def get_config(self):
    return {
        "projection_dim": self._projection_dim,
        "diag_scale": self._diag_scale,
        "use_bias": self._use_bias,
        "preactivation": self._preactivation_cfg if (self._preactivation_cfg is None or isinstance(self._preactivation_cfg, str))
                         else getattr(self._preactivation_cfg, "__name__", str(self._preactivation_cfg)),
        "kernel_initializer": self._kernel_initializer if isinstance(self._kernel_initializer, str) else "custom",
        "bias_initializer": self._bias_initializer if isinstance(self._bias_initializer, str) else "custom",
        "kernel_regularizer": None if self._kernel_regularizer is None else getattr(self._kernel_regularizer, "__name__", "custom"),
        "bias_regularizer": None if self._bias_regularizer is None else getattr(self._bias_regularizer, "__name__", "custom"),
        "name": self.name,
    }

  @classmethod
  def from_config(cls, config):
    cfg = dict(config)
    cfg.pop("kernel_regularizer", None); cfg.pop("bias_regularizer", None)
    return cls(**cfg)
