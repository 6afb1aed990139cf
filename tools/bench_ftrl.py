"""FTRL (K12) call times and achieved HBM bandwidth.

    python tools/bench_ftrl.py [--quick] [--out PATH]

Sparse legs: one table per call, batch n = 16384 ids (the cfg3 batch), d = 64, tables of 10M and 1M rows, ids uniform
and Zipf(1.05).  Dense leg: one multi-tensor call over the parameters of cfg5's full-rank Cross (845 x 845 + 845) and top
MLP (845 -> 512 -> 256 -> 1).  Every leg runs in both power modes: lr_power = -0.5 (sqrt, the default) and
lr_power = -0.3 (fp64 pow).  Two times per leg, both from CUDA events after warm-up calls of the same shape, the median
of three windows of at least 0.2 s each, with the spread over the windows:
  seconds        back-to-back calls through ops (host checks and the ctypes call included); four id batches rotate
  graph_seconds  the device time alone: the four calls (one per batch) captured in one CUDA graph and replayed, per call
Algorithmic bytes (csrc/ftrl.cu): sparse 6*u*d*4 + n*d*4 with u the unique in-range ids of the batch; dense 7*N*4.  The
fraction is of the H100 SXM data-sheet bandwidth, 3.35 TB/s, at the graph time.  The card's name and power limit are
read (not changed) in the same run.
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from recommenders_b200 import ops  # noqa: E402
from bench_adam import card, timed  # noqa: E402

HBM_DATASHEET = 3.35e12
MODES = {"sqrt": -0.5, "pow": -0.3}


def _rule(lr_power):
  lr = 0.05
  return dict(lr=lr, lr_power=lr_power, l1=1e-3, l2a=ops.ftrl_l2(1e-3, 0.0, lr), l2_shrinkage=0.0)


def graph_timed(fn, calls_in_fn):
  """Seconds per call of `fn` (which makes `calls_in_fn` calls) captured in one CUDA graph and replayed."""
  fn(); torch.cuda.synchronize()
  gr = torch.cuda.CUDAGraph()
  with torch.cuda.graph(gr):
    fn()
  sec, spread, _ = timed(gr.replay)
  return sec / calls_in_fn, spread


def _leg(sec, spread, calls, gsec, gspread, by):
  return {"seconds": sec, "spread": spread, "calls_per_window": calls, "graph_seconds": gsec, "graph_spread": gspread,
          "algorithmic_bytes": by, "GBps": by / gsec / 1e9, "frac_of_3.35TBps": by / gsec / HBM_DATASHEET}


def sparse_legs(quick, dev):
  out = {}
  n, d = 16384, 64
  g = torch.Generator(device=dev); g.manual_seed(3)
  rng = np.random.RandomState(5)
  for rows in ((1_000_000,) if quick else (10_000_000, 1_000_000)):
    table = (torch.rand((rows, d), generator=g, device=dev) - 0.5) * 0.1
    acc = torch.full_like(table, 0.1); lin = torch.zeros_like(table)
    grads = torch.randn((n, d), generator=g, device=dev) * 0.01
    batches = {"uniform": [torch.randint(0, rows, (n,), generator=g, device=dev) for _ in range(4)],
               "zipf": [torch.from_numpy(np.minimum(rng.zipf(1.05, size=n) - 1, rows - 1)).to(dev) for _ in range(4)]}
    for kind, ids in batches.items():
      u = float(np.mean([torch.unique(i).numel() for i in ids]))
      for mode, lr_power in MODES.items():
        rule = _rule(lr_power)
        it = [0]

        def call():
          it[0] += 1
          ops.sparse_ftrl_(table, acc, lin, ids[it[0] % 4], grads, **rule)
        sec, spread, calls = timed(call)
        gsec, gspread = graph_timed(lambda: [ops.sparse_ftrl_(table, acc, lin, i, grads, **rule) for i in ids], len(ids))
        out[f"{rows // 1_000_000}M_x{d}_{kind}_{mode}"] = dict(
            _leg(sec, spread, calls, gsec, gspread, 6 * u * d * 4 + n * d * 4), unique_rows=u)
    del table, acc, lin, grads, batches
    torch.cuda.empty_cache()
  return out


def dense_legs(dev):
  shapes = [(845, 845), (845,), (845, 512), (512,), (512, 256), (256,), (256, 1), (1,)]
  g = torch.Generator(device=dev); g.manual_seed(4)
  xs = [torch.randn(s, generator=g, device=dev) * 0.05 for s in shapes]
  gs = [torch.randn(s, generator=g, device=dev) * 0.01 for s in shapes]
  accs = [torch.full(s, 0.1, device=dev) for s in shapes]
  lins = [torch.zeros(s, device=dev) for s in shapes]
  N = sum(x.numel() for x in xs)
  out = {}
  for mode, lr_power in MODES.items():
    rule = _rule(lr_power)
    call = lambda: ops.ftrl_dense_(xs, gs, accs, lins, **rule)
    sec, spread, calls = timed(call)
    gsec, gspread = graph_timed(call, 1)
    out[mode] = dict(_leg(sec, spread, calls, gsec, gspread, 7 * N * 4), elements=N, variables=len(shapes),
                     shapes="cfg5 Cross 845x845 + 845, top MLP 845->512->256->1")
  return out


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--quick", action="store_true", help="the 1M-row table only")
  ap.add_argument("--out", default=None)
  a = ap.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit("bench_ftrl.py needs a CUDA device")
  dev = torch.device("cuda", 0)
  res = {"card": card(), "sparse": sparse_legs(a.quick, dev), "dense": dense_legs(dev)}
  res["card_after"] = card()
  line = json.dumps(res)
  print(line)
  if a.out:
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as fh:
      fh.write(line + "\n")


if __name__ == "__main__":
  main()
