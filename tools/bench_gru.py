"""Times K19, tf-keras `GRU` on the device (ops.gru), next to torch.nn.GRU (cuDNN, fp32, TF32 off) in the same run.

    python tools/bench_gru.py [--windows 5] [--calls 10] [--out profiles/h100_gru.json]

Shapes (B, T, D, u): the sequential retrieval tutorial's query tower (12800, 10, 32, 32), then (4096, 50, 64, 128),
(1024, 200, 256, 256) and (256, 20, 1024, 1024).  Per shape:
  - forward: ops.gru under no_grad (the K6 projection and the K19 recurrence), and cuDNN's forward under no_grad;
  - forward + backward: the same with every weight, x and h_0 requiring gradients, backward from a fixed h_T gradient;
  - the recurrence kernel alone (tfrs_gru_fwd_f32 on a precomputed projection, nothing saved), with its FLOP/s:
    6 u^2 per row and step for h.U (multiply-adds counted as two) over kernel time, against the H100 SXM data sheet's
    67 TFLOP/s FP32 (a bound for a 700 W card; the share is of that figure, not of a measured peak).
Device time per call: CUDA events around `calls` back-to-back calls after a warm-up, in several windows; the median
with the spread.  The outputs of both implementations are compared on the same weights.  The card's name and power limit
are read in the same run."""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from recommenders_b200 import ops  # noqa: E402

FP32_FLOPS = 67e12
SHAPES = [(12800, 10, 32, 32), (4096, 50, 64, 128), (1024, 200, 256, 256), (256, 20, 1024, 1024)]


def _card():
  name = torch.cuda.get_device_name()
  try:
    q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,enforced.power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
    power = q[torch.cuda.current_device()] if q else "unknown"
  except (OSError, subprocess.SubprocessError):
    power = "unknown"
  return {"name": name, "power_limit_enforced_limit_max_sm_clock": power}


def _windows(fn, windows, calls):
  for _ in range(2):
    fn()
  torch.cuda.synchronize()
  per = []
  for _ in range(windows):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(calls):
      fn()
    b.record()
    b.synchronize()
    per.append(a.elapsed_time(b) * 1e3 / calls)
  return {"us_median": round(statistics.median(per), 2), "us_min": round(min(per), 2), "us_max": round(max(per), 2)}


def _to_torch(a, u):
  """Keras columns (z, r, h) -> torch.nn.GRU rows (r, z, n)."""
  return torch.cat([a[..., u:2 * u], a[..., :u], a[..., 2 * u:]], -1).T.contiguous()


def bench_shape(B, T, D, u, windows, calls):
  g = torch.Generator(device="cuda").manual_seed(B + T + D + u)
  x = torch.randn((B, T, D), device="cuda", generator=g)
  W = (torch.rand((D, 3 * u), device="cuda", generator=g) * 2 - 1) * (6 / (D + 3 * u)) ** 0.5
  U = torch.randn((u, 3 * u), device="cuda", generator=g) / u ** 0.5
  bias = torch.randn((2, 3 * u), device="cuda", generator=g) * 0.1
  h0 = torch.rand((B, u), device="cuda", generator=g) * 2 - 1
  gh = torch.randn((B, u), device="cuda", generator=g)
  net = torch.nn.GRU(D, u, batch_first=True).cuda()
  with torch.no_grad():
    net.weight_ih_l0.copy_(_to_torch(W, u)); net.weight_hh_l0.copy_(_to_torch(U, u))
    net.bias_ih_l0.copy_(_to_torch(bias[0], u)); net.bias_hh_l0.copy_(_to_torch(bias[1], u))
  leaves = [t.clone().requires_grad_() for t in (x, W, U, bias, h0)]
  xg, hg = leaves[0], leaves[4].detach().clone().requires_grad_()

  def ours_fwd():
    with torch.no_grad():
      return ops.gru(x, W, U, bias, h0)[1]

  def ours_step():
    for t in leaves:
      t.grad = None
    _, h = ops.gru(*leaves)
    h.backward(gh)

  def cudnn_fwd():
    with torch.no_grad():
      return net(x, h0[None])[1][0]

  def cudnn_step():
    xg.grad = None; hg.grad = None; net.zero_grad(set_to_none=True)
    net(xg, hg[None])[1][0].backward(gh)

  with torch.no_grad():
    gx = ops.dense(x.reshape(B * T, D), W, bias[0]).reshape(B, T, 3 * u)
  kernel = lambda: ops._gru_fwd(gx, U, bias[1], h0, None, 0, False, False)
  diff = (ours_fwd() - cudnn_fwd()).abs().max().item()
  rec = _windows(kernel, windows, calls)
  flops = 6.0 * B * T * u * u
  rec["tflops"] = round(flops / (rec["us_median"] * 1e-6) / 1e12, 3)
  rec["share_of_67TFLOPs_fp32"] = round(flops / (rec["us_median"] * 1e-6) / FP32_FLOPS, 4)
  row = {"B": B, "T": T, "D": D, "units": u,
         "ours_fwd": _windows(ours_fwd, windows, calls), "cudnn_fwd": _windows(cudnn_fwd, windows, calls),
         "ours_fwd_bwd": _windows(ours_step, windows, calls), "cudnn_fwd_bwd": _windows(cudnn_step, windows, calls),
         "recurrence_kernel_fwd": rec, "max_abs_diff_h_T_vs_cudnn": diff}
  row["fwd_speedup_vs_cudnn"] = round(row["cudnn_fwd"]["us_median"] / row["ours_fwd"]["us_median"], 3)
  row["fwd_bwd_speedup_vs_cudnn"] = round(row["cudnn_fwd_bwd"]["us_median"] / row["ours_fwd_bwd"]["us_median"], 3)
  return row


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--windows", type=int, default=5)
  ap.add_argument("--calls", type=int, default=10)
  ap.add_argument("--out", default=None)
  args = ap.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit("bench_gru needs a CUDA device; no number is measured without one")
  torch.backends.cuda.matmul.allow_tf32 = False
  torch.backends.cudnn.allow_tf32 = False
  torch.backends.cudnn.enabled = True
  out = {"card": _card(), "windows": args.windows, "calls_per_window": args.calls,
         "cudnn": torch.backends.cudnn.version(), "rows": [bench_shape(*s, args.windows, args.calls) for s in SHAPES]}
  text = json.dumps(out, indent=1)
  print(text)
  if args.out:
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as fh:
      fh.write(text + "\n")


if __name__ == "__main__":
  main()
