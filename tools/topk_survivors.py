"""Survivors, records, retries and fallbacks per query of one tensor-core top-K call on a bench.py workload.

    python tools/topk_survivors.py [--workload cfg2] [--batches 1]

Corpus and queries are bench.py's (N(0, 1), seeds 1 / 2; query batch j is the j-th of the generator).  After each call
the per-row state is read out of the call's workspace at the offsets tfrs_topk_tc_layout and tfrs_topk_tc_retry_layout
report:
  survivors  screening scores >= the row's filter threshold in its octet records (what the select kernel ranks)
  records    octet records in its survivor lists (what the filter pass stored)
  retries    rows filtered again at the guaranteed threshold (the k-th bin bound)
  fallbacks  rows that took the exact CUDA-core scan
Prints one JSON line per batch.
"""
import argparse
import ctypes
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from bench import WORKLOADS, gen_corpus_block  # noqa: E402
from recommenders_b200 import ops  # noqa: E402


def row_state(Q, N, d, k):
  lay = (ctypes.c_int64 * 10)()
  ops.check(ops.lib().tfrs_topk_tc_layout(Q, N, d, k, lay), "topk_tc_layout")
  o_count, o_ovf, o_thr, o_cand, segs, cap, Qp = [int(x) for x in lay[:7]]
  rl = (ctypes.c_int64 * 4)()
  ops.check(ops.lib().tfrs_topk_tc_retry_layout(Q, N, d, k, rl), "topk_tc_retry_layout")
  o_retry, k_filter = int(rl[1]), int(rl[2])
  dev = torch.device("cuda", torch.cuda.current_device())
  ws = ops.workspace(0, dev, "tc")
  base = (-ws.data_ptr()) % 16
  torch.cuda.synchronize()

  def arr(off, n, dtype):
    return ws[base + off: base + off + 4 * n].view(dtype)

  count = arr(o_count, Qp * segs, torch.int32).view(Qp, segs)[:Q].to(torch.int64).clamp(max=cap)
  thr = arr(o_thr, Q, torch.float32)
  cand_s = arr(o_cand, Qp * segs * cap * 8, torch.float32).view(Qp, segs, cap, 8)[:Q]
  cand_i = arr(o_cand + Qp * segs * cap * 32, Qp * segs * cap, torch.int32).view(Qp, segs, cap)[:Q]
  live = torch.arange(cap, device=dev)[None, None, :] < count[:, :, None]
  col = cand_i.to(torch.int64)[..., None] + torch.arange(8, device=dev)
  surv = ((cand_s >= thr[:, None, None, None]) & live[..., None] & (col < N)).flatten(1).sum(1)
  return {"k_filter": k_filter, "survivors": surv, "records": count.sum(1),
          "retries": int((arr(o_retry, Q, torch.int32) != 0).sum()), "fallbacks": int((arr(o_ovf, Q, torch.int32) != 0).sum())}


def stats(t):
  t = t.double()
  return {"mean": round(float(t.mean()), 1), "p50": float(t.median()), "max": int(t.max())}


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--workload", default="cfg2", choices=sorted(WORKLOADS))
  ap.add_argument("--batches", type=int, default=1)
  args = ap.parse_args()
  N, d, Q, k = WORKLOADS[args.workload]
  dev = torch.device("cuda", 0)
  torch.cuda.set_device(dev)
  c = torch.cat([gen_corpus_block(torch, dev, b0, min(1_000_000, N - b0), d) for b0 in range(0, N, 1_000_000)], 0)
  g = torch.Generator(device=dev); g.manual_seed(2)
  idx = ops.index_build(c)
  for j in range(args.batches):
    q = torch.randn((Q, d), generator=g, device=dev)
    ops.topk_tc(q, c, idx, k)
    st = row_state(Q, N, d, k)
    print(json.dumps({"workload": args.workload, "batch": j, "gpu": torch.cuda.get_device_name(dev), "k": k,
                      "k_filter": st["k_filter"], "survivors": stats(st["survivors"]), "records": stats(st["records"]),
                      "retries": st["retries"], "fallbacks": st["fallbacks"]}), flush=True)


if __name__ == "__main__":
  sys.exit(main())
