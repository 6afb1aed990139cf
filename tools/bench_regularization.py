"""Times K23 (ops.dropout) and K24 (ops.batch_norm in training) on the device, next to torch's F.dropout and
F.batch_norm(training=True) on the same inputs in the same run.

    python tools/bench_regularization.py [--windows 5] [--calls 20] [--out profiles/h100_regularization.json]

Dropout shapes: a SASRec activation (256, 200, 64), an MLP activation (8192, 1024) and 2^26 elements; rate 0.2, the
forward (the backward is the same kernel on dy).  Batch norm shapes (N, d): (8192, 256), (65536, 1024) and (256*200, 64)
with a padding mask (ours only: torch's batch_norm has no mask, so its row for that shape runs unmasked); the training
forward (moving statistics updated) and the forward + backward (x, gamma and beta requiring gradients).
Three times per call, all after a warm-up:
  * events: CUDA events around `calls` back-to-back calls, in several windows; the median with the spread (bench_gru's
    helpers).  Where the host cannot keep the device busy this is host time, not device time;
  * device: the sum of the durations torch.profiler records on the device (kernels, memsets, copies) over `calls` calls,
    divided by `calls`; no host time;
  * host: wall clock around `calls` calls with no synchronisation inside, divided by `calls`: the cost of issuing a
    call (Python, ctypes or torch dispatch, autograd, launches) while the device keeps up.
The speedups are taken from the device times.  GB/s counts the bytes the algorithm needs: dropout reads x and writes y (8 B per
element); the batch-norm forward reads x twice and writes y (12 B per element), the backward reads x and dy twice and
writes dx (20 B per element).  The card's name and power limit are read in the same run."""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from bench_gru import _card, _windows  # noqa: E402
from recommenders_b200 import ops  # noqa: E402

DROPOUT_SHAPES = [("sasrec", (256, 200, 64)), ("mlp", (8192, 1024)), ("2^26", (1 << 26,))]
BN_SHAPES = [("mlp_256", 8192, 256, None), ("mlp_1024", 65536, 1024, None), ("sasrec_masked", 256 * 200, 64, (256, 200))]
RATE = 0.2


def _device_us(fn, calls):
  fn()
  torch.cuda.synchronize()
  with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
    for _ in range(calls):
      fn()
    torch.cuda.synchronize()
  total = sum(e.time_range.elapsed_us() for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA)
  if total <= 0:
    raise RuntimeError("torch.profiler recorded no device activity; no device time is measured")
  return round(total / calls, 2)


def _host_us(fn, calls):
  fn()
  torch.cuda.synchronize()
  t = time.perf_counter()
  for _ in range(calls):
    fn()
  dt = time.perf_counter() - t
  torch.cuda.synchronize()
  return round(dt * 1e6 / calls, 2)


def _timed(row, key, fn, windows, calls):
  row[key] = _windows(fn, windows, calls)
  row[key + "_device_us"] = _device_us(fn, calls)
  row[key + "_host_us"] = _host_us(fn, calls)


def _gbps(nbytes, us):
  return round(nbytes / (us * 1e-6) / 1e9, 1)


def bench_dropout(name, shape, windows, calls):
  g = torch.Generator(device="cuda").manual_seed(len(shape))
  x = torch.randn(shape, device="cuda", generator=g)
  n = x.numel()
  state = {"call": 0}

  def ours():
    state["call"] += 1
    return ops.dropout(x, RATE, 12345, state["call"])

  def theirs():
    return F.dropout(x, RATE, training=True)

  kept = float((ours() != 0).float().mean())
  row = {"shape": name, "dims": list(shape), "elements": n, "rate": RATE, "ours_keep_fraction": round(kept, 5),
         "floor_us_at_3.35TBps": round(8 * n / 3.35e12 * 1e6, 1)}
  _timed(row, "ours", ours, windows, calls)
  _timed(row, "torch_dropout", theirs, windows, calls)
  row["ours_GBps"] = _gbps(8 * n, row["ours_device_us"])
  row["torch_GBps"] = _gbps(8 * n, row["torch_dropout_device_us"])
  row["device_speedup_vs_torch"] = round(row["torch_dropout_device_us"] / row["ours_device_us"], 3)
  return row


def bench_batch_norm(name, N, d, mask_bt, windows, calls):
  g = torch.Generator(device="cuda").manual_seed(N + d)
  x = torch.randn((N, d), device="cuda", generator=g) * 2 + 1
  dy = torch.randn((N, d), device="cuda", generator=g)
  gamma, beta = torch.randn(d, device="cuda", generator=g), torch.randn(d, device="cuda", generator=g)
  mask = None
  if mask_bt is not None:
    B, T = mask_bt
    lengths = torch.randint(1, T + 1, (B, 1), device="cuda", generator=g)
    mask = (torch.arange(T, device="cuda")[None] < lengths).reshape(N)
  mm, mv = torch.zeros(d, device="cuda"), torch.ones(d, device="cuda")
  tmm, tmv = mm.clone(), mv.clone()
  leaves = [t.clone().requires_grad_() for t in (x, gamma, beta)]
  tleaves = [t.clone().requires_grad_() for t in (x, gamma, beta)]

  def ours_fwd():
    with torch.no_grad():
      return ops.batch_norm(x, gamma, beta, mm, mv, True, 0.99, 1e-3, mask)

  def ours_step():
    for t in leaves:
      t.grad = None
    ops.batch_norm(*leaves, mm, mv, True, 0.99, 1e-3, mask).backward(dy)

  def torch_fwd():
    with torch.no_grad():
      return F.batch_norm(x, tmm, tmv, gamma, beta, training=True, momentum=0.01, eps=1e-3)

  def torch_step():
    for t in tleaves:
      t.grad = None
    F.batch_norm(tleaves[0], tmm, tmv, tleaves[1], tleaves[2], training=True, momentum=0.01, eps=1e-3).backward(dy)

  row = {"shape": name, "N": N, "d": d, "mask": "padding (ours only)" if mask is not None else None}
  for key, fn in (("ours_fwd", ours_fwd), ("torch_fwd", torch_fwd), ("ours_fwd_bwd", ours_step),
                  ("torch_fwd_bwd", torch_step)):
    _timed(row, key, fn, windows, calls)
  if mask is None:
    row["max_abs_diff_y_vs_torch"] = (ours_fwd() - torch_fwd()).abs().max().item()
  e = N * d
  for key, nbytes in (("ours_fwd", 12 * e), ("torch_fwd", 12 * e), ("ours_fwd_bwd", 32 * e), ("torch_fwd_bwd", 32 * e)):
    row[key + "_GBps"] = _gbps(nbytes, row[key + "_device_us"])
  row["fwd_device_speedup_vs_torch"] = round(row["torch_fwd_device_us"] / row["ours_fwd_device_us"], 3)
  row["fwd_bwd_device_speedup_vs_torch"] = round(row["torch_fwd_bwd_device_us"] / row["ours_fwd_bwd_device_us"], 3)
  return row


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--windows", type=int, default=5)
  ap.add_argument("--calls", type=int, default=20)
  ap.add_argument("--out", default=None)
  args = ap.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit("bench_regularization needs a CUDA device; no number is measured without one")
  out = {"card": _card(), "windows": args.windows, "calls_per_window": args.calls,
         "dropout": [bench_dropout(n, s, args.windows, args.calls) for n, s in DROPOUT_SHAPES],
         "batch_norm": [bench_batch_norm(*s, args.windows, args.calls) for s in BN_SHAPES]}
  text = json.dumps(out, indent=1)
  print(text)
  if args.out:
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as fh:
      fh.write(text + "\n")


if __name__ == "__main__":
  main()
