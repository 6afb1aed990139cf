"""Multi-interest (maxsim) retrieval: queries/s of BruteForce with [Q, H, d] queries, and where the time goes.

    python tools/bench_maxsim.py [--n 1000000] [--q 4096] [--heads 1,2,4,8] [--out profiles/h100_maxsim.json]

Corpus: bench.py's cfg2 data (d = 64, N(0, 1) rows in 1M-row blocks seeded 1 + first row); queries N(0, 1) [Q, H, 64]
from seed 2; k = 100.  For every H it times, each with CUDA events after warm-up calls of the same shape (the median of
three windows of at least 0.2 s each, with the spread over the windows):
  step   BruteForce.call on the [Q, H, d] queries (what a user runs)
  scan   the per-head top-100 of the Q*H head rows alone, in the chunks ops.topk_maxsim uses
  merge  K26 alone, on those [Q, H, 100] lists
  2d     BruteForce.call on the same Q*H head rows as a [Q*H, d] batch: the 2-D step the scan part should cost
It checks that the step's result equals the merge of the timed scan's lists, and at H = 1 that it equals the 2-D call
bit for bit.  The card's name and power limit are read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from recommenders_b200 import ops  # noqa: E402
from recommenders_b200.layers.factorized_top_k import BruteForce  # noqa: E402

D, K = 64, 100


def card():
  fields = ["name", "power.limit", "enforced.power.limit", "clocks.max.sm"]
  out = subprocess.run(["nvidia-smi", f"--query-gpu={','.join(fields)}", "--format=csv,noheader,nounits"],
                       capture_output=True, text=True)
  return dict(zip(fields, [s.strip() for s in out.stdout.splitlines()[0].split(",")]))


def corpus(N, dev):
  x = torch.empty((N, D), device=dev)
  g = torch.Generator(device=dev)
  for b0 in range(0, N, 1_000_000):
    g.manual_seed(1 + b0)
    x[b0:b0 + 1_000_000] = torch.randn((min(1_000_000, N - b0), D), generator=g, device=dev)
  return x


def timed(fn, windows=3, min_window_s=0.2, warm=2):
  """Seconds per call: the median of `windows` CUDA-event windows, each of at least `min_window_s` of work (the call
  count is set from the warm-up), and the (min, max) spread over the windows."""
  torch.cuda.synchronize(); t0 = time.perf_counter()
  for _ in range(warm):
    fn()
  torch.cuda.synchronize()
  reps = max(1, int(min_window_s / max((time.perf_counter() - t0) / warm, 1e-6)) + 1)
  per = []
  for _ in range(windows):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
      fn()
    b.record()
    torch.cuda.synchronize()
    per.append(a.elapsed_time(b) / reps / 1e3)
  per.sort()
  return per[len(per) // 2], (per[0], per[-1]), reps


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--n", type=int, default=1_000_000)
  ap.add_argument("--q", type=int, default=4096)
  ap.add_argument("--heads", default="1,2,4,8")
  ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_maxsim.json"))
  args = ap.parse_args()
  assert torch.cuda.is_available(), "bench_maxsim measures on a CUDA device"
  dev = torch.device("cuda", 0)
  N, Q = args.n, args.q
  x = corpus(N, dev)
  bf = BruteForce(k=K).index(x)
  info = {"card": card(), "N": N, "d": D, "k": K, "Q": Q, "tensor_core_scan": bf._tc_index is not None, "rows": []}
  for H in [int(s) for s in args.heads.split(",")]:
    g = torch.Generator(device=dev)
    g.manual_seed(2)
    q3 = torch.randn((Q, H, D), generator=g, device=dev)
    rows = q3.reshape(Q * H, D)
    step = max(1, ops.TC_MAX_Q_PER_CALL // H)
    lists_s = torch.empty((Q * H, K), device=dev)
    lists_i = torch.empty((Q * H, K), dtype=torch.int64, device=dev)

    def scan():
      for lo in range(0, Q, step):
        hi = min(Q, lo + step)
        ops.topk(rows[lo * H:hi * H], x, K, image=bf._tc_index, out=(lists_s[lo * H:hi * H], lists_i[lo * H:hi * H]))

    def merge():
      return ops.maxsim_merge(lists_s.view(Q, H, K), lists_i.view(Q, H, K), K)

    scan()
    got_s, got_i = bf(q3)
    ms, mi = merge()
    assert torch.equal(got_i.to(torch.int64), mi) and torch.equal(got_s.view(torch.int32), ms.view(torch.int32))
    if H == 1:
      s2, i2 = bf(rows)
      assert torch.equal(got_i, i2) and torch.equal(got_s.view(torch.int32), s2.view(torch.int32))
    t_step, sp_step, r_step = timed(lambda: bf(q3))
    t_scan, sp_scan, _ = timed(scan)
    t_merge, sp_merge, _ = timed(merge)
    t_2d, sp_2d, _ = timed(lambda: bf(rows))
    row = {"H": H, "head_rows": Q * H, "queries_per_s": Q / t_step,
           "queries_per_s_spread": [Q / sp_step[1], Q / sp_step[0]], "calls_per_window": r_step,
           "step_ms": t_step * 1e3, "scan_ms": t_scan * 1e3, "merge_ms": t_merge * 1e3, "2d_same_rows_ms": t_2d * 1e3,
           "step_ms_spread": [sp_step[0] * 1e3, sp_step[1] * 1e3], "scan_ms_spread": [sp_scan[0] * 1e3, sp_scan[1] * 1e3],
           "merge_ms_spread": [sp_merge[0] * 1e3, sp_merge[1] * 1e3], "2d_ms_spread": [sp_2d[0] * 1e3, sp_2d[1] * 1e3],
           "merge_share_of_step": t_merge / t_step, "scan_over_2d": t_scan / t_2d}
    info["rows"].append(row)
    print(json.dumps(row), flush=True)
    del q3, rows, lists_s, lists_i
    torch.cuda.empty_cache()
  print(json.dumps(info["card"]))
  os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
  with open(args.out, "w") as fh:
    json.dump(info, fh, indent=1)


if __name__ == "__main__":
  main()
