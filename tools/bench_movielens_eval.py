"""Users/s of `examples.movielens.evaluate`'s device pass (`ops.topk_overriding` + `ops.count_listed`) on synthetic
MovieLens-shaped data.

    python tools/bench_movielens_eval.py [--shapes ml-1m,ml-25m] [--k 10] [--d 64] [--reps 5] [--out FILE]

Shapes: ml-1m = 6040 users x 3706 movies, ml-25m = 162541 users x 62423 movies.  Watch histories are skewed like the
real sets (a log-normal with the ML-1M / ML-25M medians and a long tail, at least 20 movies per user), so every run
has users on both routes; the JSON line gives the share of users on each route.  Test lists hold 10 entries per user.
The timed window is the device pass only, from embeddings and host CSR lists already built, ended by a synchronise;
the host-side list building of `evaluate` is timed separately.  Prints one JSON line per shape, with the GPU's name and
power limit read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from recommenders_b200 import ops  # noqa: E402
from recommenders_b200.examples import movielens  # noqa: E402

SHAPES = {"ml-1m": (6040, 3706, 96.0), "ml-25m": (162541, 62423, 71.0)}   # users, movies, median history


def _histories(rng, U, N, median):
  h = np.exp(rng.normal(np.log(median), 1.0, U)).astype(np.int64)
  return np.clip(h, 20, N - 1)


def _csr(rng, lengths, N, unique):
  owner = np.repeat(np.arange(len(lengths)), lengths)
  rows = rng.randint(0, N, owner.size).astype(np.int64)
  if unique:
    key = np.unique(owner * N + rows)
    owner, rows = key // N, key % N
  off = np.zeros(len(lengths) + 1, np.int64)
  np.cumsum(np.bincount(owner, minlength=len(lengths)), out=off[1:])
  return off, rows


def _gpu():
  try:
    pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                        capture_output=True, text=True, timeout=30).stdout.strip()
  except (OSError, subprocess.SubprocessError):
    pl = "unknown"
  return torch.cuda.get_device_name(0), pl


def run(shape, k, d, reps, seed=0):
  U, N, median = SHAPES[shape]
  rng = np.random.RandomState(seed)
  dev = torch.device("cuda", 0)
  users = torch.from_numpy(rng.normal(size=(U, d)).astype(np.float32)).to(dev)
  movies = torch.from_numpy(rng.normal(size=(N, d)).astype(np.float32)).to(dev)
  hist = _histories(rng, U, N, median)
  tr_off, tr_rows = _csr(rng, hist, N, unique=True)
  te_off, te_rows = _csr(rng, np.full(U, 10), N, unique=False)
  width = ops.override_width(k, np.diff(tr_off), N)

  # host side of evaluate on the same lists (user ids 0..U-1, movie ids 0..N-1)
  t0 = time.perf_counter()
  movielens.evaluation_lists(np.arange(N), {"user_id": np.repeat(np.arange(U), 10), "movie_id": te_rows},
                             {"user_id": np.repeat(np.arange(U), np.diff(tr_off)), "movie_id": tr_rows})
  host_s = time.perf_counter() - t0

  image = ops.index_build(movies) if N >= ops.TC_MIN_N else None
  def step():
    _, top = ops.topk_overriding(users, movies, k, tr_off, tr_rows, image=image)
    return ops.count_listed(top, te_off, te_rows)

  step(); torch.cuda.synchronize()   # warm every width class and the workspaces
  times = []
  for _ in range(reps):
    t0 = time.perf_counter()
    step()
    torch.cuda.synchronize()
    times.append(time.perf_counter() - t0)
  name, power = _gpu()
  med = float(np.median(times))
  return {
      "shape": shape, "users": U, "movies": N, "d": d, "k": k,
      "history_median": int(np.median(hist)), "history_max": int(hist.max()),
      "scan_route_share": float((width > 0).mean()), "dense_route_share": float((width == 0).mean()),
      "tensor_core_classes": sorted(int(w) for w in np.unique(width[width > 0]) if image is not None
                                    and ops.uses_tc_scan(int((width == w).sum()), N, d, int(w))),
      "device_pass_s_median": med, "device_pass_s_min": float(min(times)), "device_pass_s_max": float(max(times)),
      "users_per_s": U / med, "host_lists_s": host_s, "gpu": name, "power_limit": power, "reps": reps,
  }


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--shapes", default="ml-1m,ml-25m")
  ap.add_argument("--k", type=int, default=10)
  ap.add_argument("--d", type=int, default=64)
  ap.add_argument("--reps", type=int, default=5)
  ap.add_argument("--out", default=None, help="also append the JSON lines to this file")
  a = ap.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit("bench_movielens_eval needs a CUDA device")
  for shape in a.shapes.split(","):
    line = json.dumps(run(shape, a.k, a.d, a.reps))
    print(line, flush=True)
    if a.out:
      with open(a.out, "a") as fh:
        fh.write(line + "\n")


if __name__ == "__main__":
  main()
