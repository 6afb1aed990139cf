"""TreeAH (K9) next to BruteForce on the same corpus: index build time and bytes, queries/s, recall@100 and LUT lookups/s.

    python tools/bench_tree_ah.py [--sizes 1000000,10000000] [--out profiles/h100_tree_ah.json]

Corpora (d = 64): "iso" is bench.py's cfg2 data (N(0,1) rows in 1M-row blocks seeded 1 + first row, queries seed 2);
"clustered" is a seeded Gaussian mixture (4096 centers N(0, 1), rows = center + 0.35 N(0, 1), queries drawn the same way).
Isotropic Gaussian rows have no cluster structure for the tree to find, so its recall there is expected to be poor; the
clustered set is the case the index is built for.  Grid: num_leaves {1000, 4000} x num_leaves_to_search {10, 40, 100} x
reordering {None, 1000}, k = 100, Q = 4096 and Q = 1.  Times come from CUDA events after warm-up calls of the same shape:
the median of three windows of at least 0.2 s each, with the spread over the windows.
LUT lookups/s = Q x (rows in the probed leaves) x B blocks / time; its bound is one int8 shared-memory lookup per lane per
clock (32 per SM per clock) at the card's maximum SM clock.
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


H100_SXM_BOOST_MHZ = 1980.0   # data-sheet maximum SM clock, used for the bound when nvidia-smi does not report one


def _num(s):
  try:
    return float(s)
  except ValueError:
    return None


def card():
  fields = ["name", "power.limit", "enforced.power.limit", "clocks.max.sm", "clocks.sm"]
  out = subprocess.run(["nvidia-smi", f"--query-gpu={','.join(fields)}", "--format=csv,noheader,nounits"],
                       capture_output=True, text=True)
  vals = dict(zip(fields, [s.strip() for s in out.stdout.splitlines()[0].split(",")]))
  clk = _num(vals["clocks.max.sm"])
  return {"nvidia_smi": vals, "sms": torch.cuda.get_device_properties(0).multi_processor_count,
          "bound_sm_clock_mhz": clk or H100_SXM_BOOST_MHZ,
          "bound_sm_clock_source": "nvidia-smi clocks.max.sm" if clk else "H100 SXM data sheet (nvidia-smi: N/A)"}


def corpus(kind, N, dev):
  if kind == "iso":
    x = torch.empty((N, D), device=dev)
    g = torch.Generator(device=dev)
    for b0 in range(0, N, 1_000_000):
      g.manual_seed(1 + b0)
      x[b0:b0 + 1_000_000] = torch.randn((min(1_000_000, N - b0), D), generator=g, device=dev)
    g.manual_seed(2)
    return x, torch.randn((4096, D), generator=g, device=dev)
  g = torch.Generator(device=dev)
  g.manual_seed(11)
  centers = torch.randn((4096, D), generator=g, device=dev)
  x = centers[torch.randint(0, 4096, (N,), generator=g, device=dev)] + 0.35 * torch.randn((N, D), generator=g, device=dev)
  q = centers[torch.randint(0, 4096, (4096,), generator=g, device=dev)] + 0.35 * torch.randn((4096, D), generator=g, device=dev)
  return x.contiguous(), q.contiguous()


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


def recall(ids, ref):
  hit = (ids.unsqueeze(2) == ref.unsqueeze(1)).any(2).float().sum(1) / ref.shape[1]
  return float(hit.mean())


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--sizes", default="1000000,10000000")
  ap.add_argument("--leaves", default="1000,4000")
  ap.add_argument("--probes", default="10,40,100")
  ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_tree_ah.json"))
  args = ap.parse_args()
  assert torch.cuda.is_available(), "bench_tree_ah measures on a CUDA device"
  dev = torch.device("cuda", 0)
  info = {"card": card(), "d": D, "k": K, "rows": []}
  bound = info["card"]["sms"] * 32 * info["card"]["bound_sm_clock_mhz"] * 1e6
  info["lut_lookup_bound_per_s"] = bound
  for N in [int(s) for s in args.sizes.split(",")]:
    for kind in ("iso", "clustered"):
      x, q = corpus(kind, N, dev)
      bf = BruteForce(k=K).index(x)
      bf_ids = bf(q)[1]
      bf_ids1 = bf(q[:1])[1]
      t4, sp4, r4 = timed(lambda: bf(q))
      t1, sp1, r1 = timed(lambda: bf(q[:1]))
      row = {"N": N, "data": kind, "impl": "BruteForce", "index_bytes": N * D * 4 + int(bf._tc_index.numel()),
             "qps_4096": 4096 / t4, "qps_4096_spread": [4096 / sp4[1], 4096 / sp4[0]], "calls_per_window_4096": r4,
             "qps_1": 1 / t1, "qps_1_spread": [1 / sp1[1], 1 / sp1[0]], "calls_per_window_1": r1, "recall_4096": 1.0}
      info["rows"].append(row); print(json.dumps(row), flush=True)
      for L in [int(s) for s in args.leaves.split(",")]:
        torch.cuda.synchronize(); t0 = time.perf_counter()
        idx = ops.tree_ah_build(x, L, 12, 2)
        torch.cuda.synchronize(); build_s = time.perf_counter() - t0
        ah_bytes = sum(int(t.numel() * t.element_size()) for t in idx.values())
        B = 32
        for P in [int(s) for s in args.probes.split(",")]:
          _, leaves = ops.topk_scan(q, idx["centroids"], P)
          sizes = (idx["leaf_offsets"][1:] - idx["leaf_offsets"][:-1]).to(torch.int64)
          probed_rows = float(sizes[leaves].sum())
          for reorder in (None, 1000):
            rows = x if reorder else None
            kp = reorder or K
            s4, sp4, r4 = timed(lambda: ops.tree_ah_search(q, idx, rows, P, K, kp))
            s1, sp1, r1 = timed(lambda: ops.tree_ah_search(q[:1], idx, rows, P, K, kp))
            ids = ops.tree_ah_search(q, idx, rows, P, K, kp)[1]
            ids1 = ops.tree_ah_search(q[:1], idx, rows, P, K, kp)[1]
            row = {"N": N, "data": kind, "impl": "TreeAH", "num_leaves": L, "num_leaves_to_search": P,
                   "num_reordering_candidates": reorder, "build_s": build_s,
                   "index_bytes": ah_bytes + (N * D * 4 if reorder else 0),
                   "qps_4096": 4096 / s4, "qps_4096_spread": [4096 / sp4[1], 4096 / sp4[0]], "calls_per_window_4096": r4,
                   "qps_1": 1 / s1, "qps_1_spread": [1 / sp1[1], 1 / sp1[0]], "calls_per_window_1": r1,
                   "recall_4096": recall(ids, bf_ids),
                   "recall_1": recall(ids1, bf_ids1), "lut_lookups_per_s_4096": probed_rows * B / s4,
                   "lut_share_of_bound_4096": probed_rows * B / s4 / bound}
            info["rows"].append(row); print(json.dumps(row), flush=True)
        del idx
      del x, q, bf
      torch.cuda.empty_cache()
  os.makedirs(os.path.dirname(args.out), exist_ok=True)
  with open(args.out, "w") as fh:
    json.dump(info, fh, indent=1)


if __name__ == "__main__":
  main()
