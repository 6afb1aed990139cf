"""Times K27, tf-keras `Conv1D` on the device (ops.conv1d), next to torch.nn.functional.conv1d (cuDNN, fp32, TF32 off) in
the same run.

    python tools/bench_conv1d.py [--windows 7] [--calls 20] [--out profiles/h100_conv1d.json]

Shapes (B, T, C -> F, k, padding, dilation): the sequential tutorial's tower width (1024, 10, 32 -> 32, 3, causal);
NextItNet blocks (256, 200, 64 -> 64, 3, causal, d = 1, 2, 4); text-CNN title encoders (1024, 30, 32 -> 64, k = 3
"same" and k = 5 "valid").  Per shape:
  - forward: both under no_grad, linear activation with a bias;
  - forward + backward: x, kernel and bias requiring gradients, backward from a fixed output gradient.
Device time per call: CUDA events around `calls` back-to-back calls after a warm-up of every shape, in several windows
that alternate between the two implementations; the median with the spread.  Keras's padding is given to cuDNN as explicit
left / right pads.  The outputs (y, dx, dW, dbias) of both are compared on the same inputs.  The card's name and power
limit are read in the same run."""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from recommenders_b200 import ops  # noqa: E402

SHAPES = [(1024, 10, 32, 32, 3, "causal", 1)] + [(256, 200, 64, 64, 3, "causal", d) for d in (1, 2, 4)] + \
         [(1024, 30, 32, 64, 3, "same", 1), (1024, 30, 32, 64, 5, "valid", 1)]


def _card():
  name = torch.cuda.get_device_name()
  try:
    q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,enforced.power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
    power = q[torch.cuda.current_device()] if q else "unknown"
  except (OSError, subprocess.SubprocessError):
    power = "unknown"
  return {"name": name, "power_limit_enforced_limit_max_sm_clock": power}


def _window(fn, calls):
  a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  a.record()
  for _ in range(calls):
    fn()
  b.record()
  b.synchronize()
  return a.elapsed_time(b) * 1e3 / calls


def _alternate(fns, windows, calls):
  """{name: median / min / max microseconds per call}, the implementations' windows interleaved."""
  per = {k: [] for k in fns}
  for _ in range(windows):
    for k, fn in fns.items():
      per[k].append(_window(fn, calls))
  return {k: {"us_median": round(statistics.median(v), 2), "us_min": round(min(v), 2), "us_max": round(max(v), 2)}
          for k, v in per.items()}


def _setup(B, T, C, F, k, padding, d):
  g = torch.Generator(device="cuda").manual_seed(B + T + C + F + k + d)
  x = torch.randn((B, T, C), device="cuda", generator=g)
  W = (torch.rand((k, C, F), device="cuda", generator=g) * 2 - 1) * (6 / (k * C + k * F)) ** 0.5
  b = torch.randn((F,), device="cuda", generator=g) * 0.1
  T_out, pl = ops.conv1d_geometry(T, k, 1, padding, d)
  pr = (T_out - 1) + d * (k - 1) + 1 - T - pl
  gy = torch.randn((B, T_out, F), device="cuda", generator=g)
  Wt = W.permute(2, 1, 0).contiguous()   # [F, C, k]
  return x, W, b, Wt, pl, pr, gy


def bench_shape(B, T, C, F, k, padding, d, windows, calls):
  x, W, b, Wt, pl, pr, gy = _setup(B, T, C, F, k, padding, d)
  leaves = [t.clone().requires_grad_() for t in (x, W, b)]
  tleaves = [t.clone().requires_grad_() for t in (x, Wt, b)]

  def torch_conv(x_, W_, b_):
    xp = torch.nn.functional.pad(x_.transpose(1, 2), (pl, pr))
    return torch.nn.functional.conv1d(xp, W_, b_, dilation=d).transpose(1, 2)

  def ours_fwd():
    with torch.no_grad():
      return ops.conv1d(x, W, b, 1, padding, d)

  def cudnn_fwd():
    with torch.no_grad():
      return torch_conv(x, Wt, b)

  def ours_step():
    for t in leaves:
      t.grad = None
    ops.conv1d(leaves[0], leaves[1], leaves[2], 1, padding, d).backward(gy)

  def cudnn_step():
    for t in tleaves:
      t.grad = None
    torch_conv(*tleaves).backward(gy)

  for fn in (ours_fwd, cudnn_fwd, ours_step, cudnn_step):   # warm-up: modules load, cuDNN picks its algorithms
    for _ in range(3):
      fn()
  torch.cuda.synchronize()
  ours_step(); cudnn_step()
  diff = {"y": (ours_fwd() - cudnn_fwd()).abs().max().item(),
          "dx": (leaves[0].grad - tleaves[0].grad).abs().max().item(),
          "dW": (leaves[1].grad - tleaves[1].grad.permute(2, 1, 0)).abs().max().item(),
          "dbias": (leaves[2].grad - tleaves[2].grad).abs().max().item()}
  fwd = _alternate({"ours": ours_fwd, "cudnn": cudnn_fwd}, windows, calls)
  step = _alternate({"ours": ours_step, "cudnn": cudnn_step}, windows, calls)
  row = {"B": B, "T": T, "C": C, "filters": F, "kernel_size": k, "padding": padding, "dilation_rate": d,
         "tensor_cores": ops.conv1d_uses_tc(B, int(gy.shape[1]), C, k, F),
         "ours_fwd": fwd["ours"], "cudnn_fwd": fwd["cudnn"], "ours_fwd_bwd": step["ours"], "cudnn_fwd_bwd": step["cudnn"],
         "max_abs_diff_vs_cudnn": diff}
  row["fwd_speedup_vs_cudnn"] = round(row["cudnn_fwd"]["us_median"] / row["ours_fwd"]["us_median"], 3)
  row["fwd_bwd_speedup_vs_cudnn"] = round(row["cudnn_fwd_bwd"]["us_median"] / row["ours_fwd_bwd"]["us_median"], 3)
  return row


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--windows", type=int, default=7)
  ap.add_argument("--calls", type=int, default=20)
  ap.add_argument("--out", default=None)
  args = ap.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit("bench_conv1d needs a CUDA device; no number is measured without one")
  torch.backends.cuda.matmul.allow_tf32 = False
  torch.backends.cudnn.allow_tf32 = False
  torch.backends.cudnn.enabled = True
  out = {"card": _card(), "windows": args.windows, "calls_per_window": args.calls, "cudnn": torch.backends.cudnn.version(),
         "rows": [bench_shape(*s, args.windows, args.calls) for s in SHAPES]}
  text = json.dumps(out, indent=1)
  print(text)
  if args.out:
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as fh:
      fh.write(text + "\n")


if __name__ == "__main__":
  main()
