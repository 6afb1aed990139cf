"""Listwise losses (K13) with fused NDCG: forward + backward times against an eager-torch restatement of the same math.

    python tools/bench_listwise.py [--quick] [--out PATH]

Shapes B x L: 8192 x 5 (the listwise_ranking tutorial's batch of 5-movie lists), 65536 x 32, 4096 x 256, 1024 x 1024.
Labels are integers 0..4 with 10 % padding; per-list weights.  One leg = one loss call with NDCG (topn = None) computed in the
same launch, plus its backward:
  fused  ops.listwise_loss(..., ndcg_stats) + backward: one K13 launch, one scaling launch (plus a 4-byte memset)
  eager  the same rules in torch ops: masked max-subtraction, sorts, cumulative sums, the [B, L, L] pair tensor for the hinge,
         NDCG by two sorts; autograd for the backward
Seconds are CUDA-event times after warm-up calls, the median of three windows of at least 0.2 s (tools/bench_adam.py timed).
Algorithmic bytes of the fused leg: pred + labels read and dl/ds written by the forward, dl/ds read and dx written by the
backward (20 B per item); the hinge also reports its pair-loop operations (B L^2 pairs) per second.  The card's name and
power limit are read (not changed) in the same run.
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

SHAPES = [(8192, 5), (65536, 32), (4096, 256), (1024, 1024)]
MODES = {"listmle": ops.LIST_LOSS_LISTMLE, "pairwise_hinge": ops.LIST_LOSS_PAIRWISE_HINGE, "softmax": ops.LIST_LOSS_SOFTMAX}


def _ndcg_eager(p, y, valid, w):
  L = p.shape[1]
  disc = ops.ndcg_discounts(p.device)[:L]
  gain = torch.where(valid, torch.exp2(y.clamp_min(0)) - 1, torch.zeros_like(y))
  pm = torch.where(valid, p, torch.full_like(p, -float("inf")))
  order = torch.sort(pm, dim=1, descending=True, stable=True).indices
  dcg = (gain.gather(1, order) * disc).sum(1)
  idcg = (torch.sort(gain, dim=1, descending=True).values * disc).sum(1)
  nd = torch.where(idcg > 0, dcg / idcg.clamp_min(1e-30), torch.zeros_like(dcg))
  return torch.stack([(w * nd).sum(), w.sum()])


def _loss_eager(mode, p, y, valid, w):
  s = p
  if mode == ops.LIST_LOSS_SOFTMAX:
    yv = torch.where(valid, y, torch.zeros_like(y))
    logits = torch.where(valid, s, torch.full_like(s, -float("inf")))
    lsm = torch.log_softmax(logits, dim=1)
    l = -(yv * torch.where(valid, lsm, torch.zeros_like(lsm))).sum(1)
  elif mode == ops.LIST_LOSS_PAIRWISE_HINGE:
    pair = valid[:, :, None] & valid[:, None, :] & (y[:, :, None] > y[:, None, :])
    h = torch.relu(1 - (s[:, :, None] - s[:, None, :]))
    cnt = pair.sum((1, 2))
    l = torch.where(pair, h, torch.zeros_like(h)).sum((1, 2)) / cnt.clamp_min(1)
  else:
    key = torch.where(valid, y + 0.5 * torch.rand_like(y), torch.full_like(y, -float("inf")))   # label desc, random ties
    order = torch.sort(key, dim=1, descending=True).indices
    ss = s.gather(1, order)
    vs = valid.gather(1, order)
    m = torch.where(vs, ss, torch.full_like(ss, -float("inf"))).amax(1, keepdim=True).clamp_min(-3e38)
    e = torch.where(vs, torch.exp(ss - m), torch.zeros_like(ss))
    S = torch.flip(torch.cumsum(torch.flip(e, [1]), 1), [1])
    l = torch.where(vs, torch.log(S.clamp_min(1e-38)) - (ss - m), torch.zeros_like(ss)).sum(1)
  return (w * l).sum() / p.shape[0]


def legs(quick):
  dev = torch.device("cuda")
  out = []
  for B, L in (SHAPES[:2] if quick else SHAPES):
    g = torch.Generator(device=dev); g.manual_seed(B + L)
    pred = torch.randn((B, L), generator=g, device=dev)
    y = torch.randint(0, 5, (B, L), generator=g, device=dev).float()
    y = torch.where(torch.rand((B, L), generator=g, device=dev) < 0.1, torch.full_like(y, -1.0), y)
    w = torch.rand((B,), generator=g, device=dev) + 0.5
    valid = y >= 0
    for name, mode in MODES.items():
      p = pred.clone().requires_grad_(True)
      stats = ops.ndcg_stats_buffer(dev)

      def fused():
        p.grad = None
        ops.listwise_loss(p, y, w, mode, ops.REDUCTION_SUM_OVER_BATCH_SIZE, 1.0, 0, 0, stats, None).backward()

      def eager():
        p.grad = None
        _loss_eager(mode, p, y, valid, w).backward()
        with torch.no_grad():
          _ndcg_eager(p, y, valid, w)

      sec, spread, calls = timed(fused)
      esec, espread, ecalls = timed(eager)
      by = 20 * B * L
      leg = {"B": B, "L": L, "loss": name, "fused_seconds": sec, "fused_spread": spread, "eager_seconds": esec,
             "eager_spread": espread, "speedup": esec / sec, "algorithmic_bytes": by, "GBps": by / sec / 1e9}
      if mode == ops.LIST_LOSS_PAIRWISE_HINGE:
        leg["pair_ops_per_second"] = B * L * L / sec
      out.append(leg)
      print(json.dumps(leg), flush=True)
      del p
    torch.cuda.empty_cache()
  return out


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--quick", action="store_true")
  ap.add_argument("--out", default=None)
  a = ap.parse_args()
  res = {"card": card(), "legs": legs(a.quick)}
  if a.out:
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as fh:
      json.dump(res, fh, indent=1)
  print(json.dumps(res["card"]))


if __name__ == "__main__":
  main()
