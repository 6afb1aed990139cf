"""Splits the time of the top-K filter pass (`tc_scan_kernel<FILTER>`, csrc/topk_tc.cu) by A/B ablation.

    python -m recommenders_b200.build --debug-switches VARIANT      # for VARIANT in full no-emit no-epilogue
    python tools/filter_probe.py [--lib NAME=PATH ...] [--workloads cfg2,cfg4] [--rounds 3] [--calls 10]

Each library (default: the three debug builds under recommenders_b200/debug/) runs in its own process, the libraries
alternate round by round, and every process times the filter stage of `--calls` calls per workload with
ops.profile_enable / profile_read (CUDA events around the stage).  Corpus and queries are bench.py's (N(0,1), seeds 1 / 2).
Prints one JSON line per (round, library) and tables of the median and range per call of the filter stage, and of the
sampled pass and finalize stages around it.

  full         the pass as built (debug switches compiled in, none set)
  no-emit      hit test and octet mask computed, no survivor record stored
  no-epilogue  the accumulators folded into one live word (meant as the MMA + bulk-TMA floor; see DEVNOTES.md)

The ablated variants stop each call after the filter pass and write no output.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
VARIANTS = ("full", "no-emit", "no-epilogue")
WORKLOADS = {"cfg2": (1_000_000, 64, 4096, 100), "cfg4": (8_000_000, 128, 4096, 100)}   # bench.py's (N, d, Q, k)


def child(args):
  sys.path.insert(0, ROOT)
  import torch
  from recommenders_b200 import ops
  dev = torch.device("cuda", 0)
  torch.cuda.set_device(dev)
  out = {"lib": os.environ.get("TFRS_B200_LIB"), "gpu": torch.cuda.get_device_name(dev)}
  for w in args.workloads.split(","):
    N, d, Q, k = WORKLOADS[w]
    blocks = []
    for b0 in range(0, N, 1_000_000):   # bench.gen_corpus_block
      g = torch.Generator(device=dev); g.manual_seed(1 + b0)
      blocks.append(torch.randn((min(1_000_000, N - b0), d), generator=g, device=dev))
    c = torch.cat(blocks, 0); del blocks
    g = torch.Generator(device=dev); g.manual_seed(2)
    q = torch.randn((Q, d), generator=g, device=dev)
    idx = ops.index_build(c)
    for _ in range(args.warmup):
      ops.topk_tc(q, c, idx, k)
    torch.cuda.synchronize()
    ops.profile_enable(True)
    for _ in range(args.calls):
      ops.topk_tc(q, c, idx, k)
    ms, calls = ops.profile_read()
    ops.profile_enable(False)
    out[w] = {"filter_ms": ms[2] / calls, "sample_ms": ms[1] / calls, "finalize_ms": ms[3] / calls, "calls": calls}
    del c, q, idx
    torch.cuda.empty_cache()
  print(json.dumps(out), flush=True)


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--lib", action="append", default=[], metavar="NAME=PATH")
  ap.add_argument("--workloads", default="cfg2,cfg4")
  ap.add_argument("--rounds", type=int, default=3)
  ap.add_argument("--calls", type=int, default=10)
  ap.add_argument("--warmup", type=int, default=3)
  ap.add_argument("--child", action="store_true", help=argparse.SUPPRESS)
  args = ap.parse_args()
  if args.child:
    return child(args)
  libs = [tuple(s.split("=", 1)) for s in args.lib] or [
      (v, os.path.join(ROOT, "recommenders_b200", "debug", f"libtfrs_b200_{v}.so")) for v in VARIANTS]
  for name, path in libs:
    if not os.path.exists(path):
      raise SystemExit(f"{name}: {path} not found (python -m recommenders_b200.build --debug-switches {name})")
  res = {name: [] for name, _ in libs}
  for r in range(args.rounds):
    for name, path in libs:
      cmd = [sys.executable, os.path.abspath(__file__), "--child", "--workloads", args.workloads,
             "--calls", str(args.calls), "--warmup", str(args.warmup)]
      p = subprocess.run(cmd, env=dict(os.environ, TFRS_B200_LIB=os.path.abspath(path)), capture_output=True, text=True)
      if p.returncode != 0:
        raise SystemExit(f"{name} failed:\n{p.stdout}\n{p.stderr}")
      line = json.loads(p.stdout.strip().splitlines()[-1])
      line.update(round=r, name=name)
      print(json.dumps(line), flush=True)
      res[name].append(line)
  for w in args.workloads.split(","):
    # the sampled pass and finalize are the same code in every variant (an ablated call does not run finalize)
    for stage in ("filter", "sample", "finalize"):
      print(f"\n{w}: {stage} stage, ms per call over {args.rounds} rounds")
      print("| variant | median | min | max |")
      print("|---|---|---|---|")
      for name, _ in libs:
        t = [x[w][stage + "_ms"] for x in res[name]]
        print(f"| {name} | {statistics.median(t):.3f} | {min(t):.3f} | {max(t):.3f} |")


if __name__ == "__main__":
  sys.exit(main())
