"""Times K20, tf-keras `LSTM` on the device (ops.lstm), next to torch.nn.LSTM (cuDNN, fp32, TF32 off) in the same run.

    python tools/bench_lstm.py [--windows 5] [--calls 10] [--out profiles/h100_lstm.json]

Shapes (B, T, D, u): tools/bench_gru.py's, the sequential retrieval tutorial's query tower (12800, 10, 32, 32) first.
Per shape:
  - forward: ops.lstm under no_grad (the K6 projection and the K20 recurrence), and cuDNN's forward under no_grad;
  - forward + backward: the same with every weight, x, h_0 and c_0 requiring gradients, backward from fixed h_T and c_T
    gradients;
  - the recurrence kernel alone (tfrs_lstm_fwd_f32 on a precomputed projection, nothing saved), with its FLOP/s:
    8 u^2 per row and step for h.U (multiply-adds counted as two) over kernel time, against the H100 SXM data sheet's
    67 TFLOP/s FP32 (a bound for a 700 W card; the share is of that figure, not of a measured peak).
Device time per call: CUDA events around `calls` back-to-back calls after a warm-up, in several windows; the median
with the spread (bench_gru's helpers).  The outputs of both implementations are compared on the same weights.  The
card's name and power limit are read in the same run."""
from __future__ import annotations

import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from bench_gru import FP32_FLOPS, SHAPES, _card, _windows  # noqa: E402
from recommenders_b200 import ops  # noqa: E402


def bench_shape(B, T, D, u, windows, calls):
  g = torch.Generator(device="cuda").manual_seed(B + T + D + u)
  x = torch.randn((B, T, D), device="cuda", generator=g)
  W = (torch.rand((D, 4 * u), device="cuda", generator=g) * 2 - 1) * (6 / (D + 4 * u)) ** 0.5
  U = torch.randn((u, 4 * u), device="cuda", generator=g) / u ** 0.5
  bias = torch.randn((4 * u,), device="cuda", generator=g) * 0.1
  h0 = torch.rand((B, u), device="cuda", generator=g) * 2 - 1
  c0 = torch.rand((B, u), device="cuda", generator=g) * 2 - 1
  gh = torch.randn((B, u), device="cuda", generator=g)
  gc = torch.randn((B, u), device="cuda", generator=g)
  # Keras's (i, f, c, o) columns are torch's (i, f, g, o) rows; Keras's one bias is b_ih with b_hh = 0
  net = torch.nn.LSTM(D, u, batch_first=True).cuda()
  with torch.no_grad():
    net.weight_ih_l0.copy_(W.T); net.weight_hh_l0.copy_(U.T)
    net.bias_ih_l0.copy_(bias); net.bias_hh_l0.zero_()
  leaves = [t.clone().requires_grad_() for t in (x, W, U, bias, h0, c0)]
  xg, hg, cg = leaves[0], leaves[4].detach().clone().requires_grad_(), leaves[5].detach().clone().requires_grad_()

  def ours_fwd():
    with torch.no_grad():
      return ops.lstm(x, W, U, bias, (h0, c0))[1]

  def ours_step():
    for t in leaves:
      t.grad = None
    _, h, c = ops.lstm(*leaves[:4], (leaves[4], leaves[5]))
    torch.autograd.backward([h, c], [gh, gc])

  def cudnn_fwd():
    with torch.no_grad():
      return net(x, (h0[None], c0[None]))[1][0][0]

  def cudnn_step():
    xg.grad = None; hg.grad = None; cg.grad = None; net.zero_grad(set_to_none=True)
    _, (h, c) = net(xg, (hg[None], cg[None]))
    torch.autograd.backward([h[0], c[0]], [gh, gc])

  with torch.no_grad():
    gx = ops.dense(x.reshape(B * T, D), W, bias).reshape(B, T, 4 * u)
  kernel = lambda: ops._lstm_fwd(gx, U, h0, c0, None, 0, False, False)
  diff = (ours_fwd() - cudnn_fwd()).abs().max().item()
  rec = _windows(kernel, windows, calls)
  flops = 8.0 * B * T * u * u
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
    raise SystemExit("bench_lstm needs a CUDA device; no number is measured without one")
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
