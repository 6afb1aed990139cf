"""TPUEmbedding's bag pooling (K11) device times and achieved HBM bandwidth, beside the K1 gather of the same rows.

    python tools/bench_embedding_bag.py [--out PATH]

Workload: a DLRM-like call of 26 tables x 64 dims (vocabularies 10^5 .. 10^6), batch B = 65536, one multi-hot feature
per table with mixed bag sizes (per table a mean hotness from {1, 2, 4, 8, 16, 32}, bag sizes uniform in
[1, 2 * mean - 1]), mean combiner, weighted; ids uniform or Zipf(1.05) over the vocabulary.
Legs, each one call captured in a CUDA graph and replayed (CUDA events, median of three windows of >= 0.2 s):
  forward   tfrs_embedding_bag_fwd_f32 over the 26 features (ids and denominators written, as under autograd)
  backward  tfrs_embedding_bag_bwd_f32 (gradient rows of every value)
  gather    tfrs_gather_f32 of the same V rows per table into [V, 64] (K1), the bound a pooled lookup is held to
Algorithmic bytes per table (V values, B bags, d = 64): forward V*(8 + 4) + V*d*4 + B*d*4 + V*8 + B*4; backward
V*(8 + 4) + V*d*4 + B*d*4 + B*4; gather V*8 + 2*V*d*4.  The fraction is of the H100 SXM data-sheet bandwidth, 3.35 TB/s.
The card's name and power limit are read (not changed) in the same run.
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

from bench_adam import card, timed  # noqa: E402
from recommenders_b200 import ops  # noqa: E402

HBM_DATASHEET = 3.35e12
TABLES, B, D = 26, 65536, 64


def workload(dev, dist, seed=0):
  rng = np.random.RandomState(seed)
  g = torch.Generator(device=dev); g.manual_seed(seed)
  feats, meta = [], []
  for t in range(TABLES):
    rows = int(10 ** (5 + t / (TABLES - 1)))
    hot = (1, 2, 4, 8, 16, 32)[t % 6]
    lens = rng.randint(1, 2 * hot, size=B)
    sp = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    V = int(sp[-1])
    ids = rng.randint(0, rows, size=V) if dist == "uniform" else np.minimum(rng.zipf(1.05, size=V) - 1, rows - 1)
    table = torch.rand((rows, D), generator=g, device=dev) - 0.5
    f = ops.BagFeature(table, torch.from_numpy(ids.astype(np.int64)).to(dev),
                       torch.empty((B, D), device=dev), torch.from_numpy(sp).to(dev),
                       torch.rand(V, generator=g, device=dev), "mean", 0, 0,
                       torch.empty(V, dtype=torch.int64, device=dev), torch.empty(B, device=dev))
    feats.append(f)
    meta.append((V, rows))
  return feats, meta


def graph_timed(fn):
  fn(); torch.cuda.synchronize()
  gr = torch.cuda.CUDAGraph()
  with torch.cuda.graph(gr):
    fn()
  return timed(gr.replay)


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--out", default=None)
  a = ap.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit("bench_embedding_bag.py needs a CUDA device")
  dev = torch.device("cuda", 0)
  res = {"card": card(), "workload": f"{TABLES} tables x {D}, B={B}, mean combiner, weighted"}
  for dist in ("uniform", "zipf"):
    feats, meta = workload(dev, dist)
    V = sum(m[0] for m in meta)
    grads = [torch.randn((B, D), device=dev) for _ in feats]
    rows = [torch.empty((m[0], D), device=dev) for m in meta]
    gath = torch.empty((max(m[0] for m in meta), D), device=dev)
    fwd = graph_timed(lambda: ops.embedding_bag(feats))
    bwd = graph_timed(lambda: ops.embedding_bag_bwd(feats, grads, rows))

    def gather_all():
      for f in feats:
        ops.gather([f.table], [f.values], out=gath[:f.values.numel()])
    gat = graph_timed(gather_all)
    by_f = sum(v * 12 + v * D * 4 + B * D * 4 + v * 8 + B * 4 for v, _ in meta)
    by_b = sum(v * 12 + v * D * 4 + B * D * 4 + B * 4 for v, _ in meta)
    by_g = sum(v * 8 + 2 * v * D * 4 for v, _ in meta)
    leg = {"values": V}
    for name, (sec, spread, calls), by in (("forward", fwd, by_f), ("backward", bwd, by_b), ("gather_K1", gat, by_g)):
      leg[name] = {"seconds": sec, "spread": spread, "calls_per_window": calls, "algorithmic_bytes": by,
                   "GBps": by / sec / 1e9, "frac_of_3.35TBps": by / sec / HBM_DATASHEET}
    leg["forward_over_gather"] = fwd[0] / gat[0]
    res[dist] = leg
    del feats, grads, rows, gath
    torch.cuda.empty_cache()
  res["card_after"] = card()
  line = json.dumps(res)
  print(line)
  if a.out:
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as fh:
      fh.write(line + "\n")


if __name__ == "__main__":
  main()
