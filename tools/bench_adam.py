"""Adam (K10) call times and achieved HBM bandwidth.

    python tools/bench_adam.py [--quick] [--out PATH]

Sparse legs: one table per call, batch n = 16384 ids (the cfg3 batch), d = 64, tables of 10M and 1M rows, ids uniform
and Zipf(1.05), not lazy (the tf-keras rule: every row decays) and lazy (touched rows only).  Dense leg: one
multi-tensor call over the parameters of cfg5's full-rank Cross (845 x 845 + 845) and top MLP (845 -> 512 -> 256 -> 1).
Times come from CUDA events around back-to-back calls after warm-up calls of the same shape: the median of three
windows of at least 0.2 s each, with the spread over the windows.  Four id batches rotate between calls.
Algorithmic bytes (csrc/adam.cu): not lazy 6*rows*d*4 + n*d*4 + rows/8; lazy 6*u*d*4 + n*d*4 with u the unique in-range
ids of the batch; dense 7*N*4.  The fraction is of the H100 SXM data-sheet bandwidth, 3.35 TB/s.  The card's name and
power limit are read (not changed) in the same run.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from recommenders_b200 import ops  # noqa: E402

HBM_DATASHEET = 3.35e12
B1, B2, EPS = 0.9, 0.999, 1e-7


def card():
  fields = ["name", "power.limit", "enforced.power.limit", "clocks.max.sm", "clocks.max.mem"]
  r = subprocess.run(["nvidia-smi", f"--query-gpu={','.join(fields)}", "--format=csv,noheader"], capture_output=True,
                     text=True)
  vals = [s.strip() for s in r.stdout.splitlines()[0].split(",")] if r.returncode == 0 and r.stdout else []
  return {"torch_name": torch.cuda.get_device_name(0), "nvidia_smi": dict(zip(fields, vals))}


def timed(fn, min_seconds=0.2, windows=3):
  """Median seconds per call over `windows` windows of at least `min_seconds`, and the spread (max - min) / median."""
  for _ in range(3):
    fn()
  torch.cuda.synchronize()
  e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  e0.record(); fn(); e1.record(); torch.cuda.synchronize()
  calls = max(5, int(min_seconds / max(e0.elapsed_time(e1) * 1e-3, 1e-6)))
  per = []
  for _ in range(windows):
    e0.record()
    for _ in range(calls):
      fn()
    e1.record()
    torch.cuda.synchronize()
    per.append(e0.elapsed_time(e1) * 1e-3 / calls)
  med = float(np.median(per))
  return med, (max(per) - min(per)) / med, calls


def sparse_legs(quick, dev):
  out = {}
  n, d = 16384, 64
  g = torch.Generator(device=dev); g.manual_seed(3)
  rng = np.random.RandomState(5)
  for rows in ((1_000_000,) if quick else (10_000_000, 1_000_000)):
    table = (torch.rand((rows, d), generator=g, device=dev) - 0.5) * 0.1
    m = torch.zeros_like(table); v = torch.zeros_like(table)
    grads = torch.randn((n, d), generator=g, device=dev) * 0.01
    batches = {"uniform": [torch.randint(0, rows, (n,), generator=g, device=dev) for _ in range(4)],
               "zipf": [torch.from_numpy(np.minimum(rng.zipf(1.05, size=n) - 1, rows - 1)).to(dev) for _ in range(4)]}
    for kind, ids in batches.items():
      u = float(np.mean([torch.unique(i).numel() for i in ids]))
      for lazy in (False, True):
        it = [0]

        def call():
          it[0] += 1
          ops.sparse_adam_(table, m, v, ids[it[0] % 4], grads, ops.adam_alpha(1e-3, B1, B2, it[0]), B1, B2, EPS, lazy=lazy)
        sec, spread, calls = timed(call)
        by = (6 * u * d * 4 + n * d * 4) if lazy else (6 * rows * d * 4 + n * d * 4 + rows / 8)
        out[f"{rows // 1_000_000}M_x{d}_{kind}_{'lazy' if lazy else 'dense_decay'}"] = {
            "seconds": sec, "spread": spread, "calls_per_window": calls, "unique_rows": u, "algorithmic_bytes": by,
            "GBps": by / sec / 1e9, "frac_of_3.35TBps": by / sec / HBM_DATASHEET}
    del table, m, v, grads, batches
    torch.cuda.empty_cache()
  return out


def dense_leg(dev):
  shapes = [(845, 845), (845,), (845, 512), (512,), (512, 256), (256,), (256, 1), (1,)]
  g = torch.Generator(device=dev); g.manual_seed(4)
  xs = [torch.randn(s, generator=g, device=dev) * 0.05 for s in shapes]
  gs = [torch.randn(s, generator=g, device=dev) * 0.01 for s in shapes]
  ms = [torch.zeros(s, device=dev) for s in shapes]
  vs = [torch.zeros(s, device=dev) for s in shapes]
  sec, spread, calls = timed(lambda: ops.adam_dense_(xs, gs, ms, vs, ops.adam_alpha(1e-3, B1, B2, 1), B1, B2, EPS))
  N = sum(x.numel() for x in xs)
  return {"seconds": sec, "spread": spread, "calls_per_window": calls, "elements": N, "variables": len(shapes),
          "algorithmic_bytes": 7 * N * 4, "GBps": 7 * N * 4 / sec / 1e9,
          "frac_of_3.35TBps": 7 * N * 4 / sec / HBM_DATASHEET,
          "shapes": "cfg5 Cross 845x845 + 845, top MLP 845->512->256->1"}


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--quick", action="store_true", help="the 1M-row table only")
  ap.add_argument("--out", default=None)
  a = ap.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit("bench_adam.py needs a CUDA device")
  dev = torch.device("cuda", 0)
  res = {"card": card(), "sparse": sparse_legs(a.quick, dev), "dense": dense_leg(dev)}
  res["card_after"] = card()
  line = json.dumps(res)
  print(line)
  if a.out:
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as fh:
      fh.write(line + "\n")


if __name__ == "__main__":
  main()
