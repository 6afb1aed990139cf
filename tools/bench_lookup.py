"""Times the K15 vocabulary lookup (layers.StringLookup / IntegerLookup) against the host mapping users write without it.

    python tools/bench_lookup.py [--windows 7] [--calls 50] [--out results.json]

Per case (IntegerLookup at V = 1M and 10M, StringLookup at V = 1M titles of 8-64 bytes; batches of 65536 ids, uniform
and Zipf(1.2), 10 % of the uniform ids outside the vocabulary):
  - device time per lookup call: CUDA events around `calls` back-to-back calls after a warm-up, in several windows;
    reported as the median with the spread, as lookups/s and as bytes/s of the modelled traffic against the H100 SXM
    data sheet's 3.35 TB/s.  Modelled bytes per value: ints 8 (value) + 4 (slot) + 8 (key) + 8 (out); strings 8 (offset)
    + len (input) + 4 (slot) + 8 (fingerprint) + 16 (key offsets) + len (key) + 8 (out); one probe each.
  - strings: host packing (pack_strings) and the one host-to-device copy, timed separately on the host clock.
  - the host alternative: a dict lookup per id in Python, np.asarray, then the upload (host clock, synchronised).
The card's name and power limit are read in the same run."""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from recommenders_b200 import ops  # noqa: E402
from recommenders_b200._strings import pack_strings, upload_packed  # noqa: E402
from recommenders_b200.layers.preprocessing import IntegerLookup, StringLookup  # noqa: E402

HBM_BYTES_PER_S = 3.35e12
B = 65536


def _card():
  name = torch.cuda.get_device_name()
  try:
    q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
    power = q[torch.cuda.current_device()] if q else "unknown"
  except (OSError, subprocess.SubprocessError):
    power = "unknown"
  return {"name": name, "power_limit_and_max_sm_clock": power}


def _windows(fn, windows, calls):
  for _ in range(3):
    fn()
  torch.cuda.synchronize()
  per = []
  for _ in range(windows):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(calls):
      fn()
    b.record()
    b.synchronize()
    per.append(a.elapsed_time(b) * 1e3 / calls)          # us per call
  return per


def _host(fn, windows, reps=3):
  fn()
  per = []
  for _ in range(windows):
    t = time.perf_counter()
    for _ in range(reps):
      fn()
    torch.cuda.synchronize()
    per.append((time.perf_counter() - t) * 1e6 / reps)
  return per


def _summary(per_us, n, nbytes=None):
  med = statistics.median(per_us)
  out = {"us_median": round(med, 2), "us_min": round(min(per_us), 2), "us_max": round(max(per_us), 2),
         "lookups_per_s": n / (med * 1e-6)}
  if nbytes is not None:
    out["modelled_bytes"] = int(nbytes)
    out["bytes_per_s"] = nbytes / (med * 1e-6)
    out["share_of_3.35TB/s"] = round(nbytes / (med * 1e-6) / HBM_BYTES_PER_S, 4)
  return out


def _batches(rng, V):
  uniform = rng.randint(0, V, size=B)
  oov = rng.rand(B) < 0.1
  zipf = (rng.zipf(1.2, size=B) - 1) % V
  return {"uniform": (uniform, oov), "zipf": (zipf, np.zeros(B, bool))}


def bench_int(V, args, rng):
  vocab = rng.permutation(np.unique(rng.randint(-2**62, 2**62, size=V + V // 8, dtype=np.int64)))[:V]
  layer = IntegerLookup(vocabulary=torch.from_numpy(vocab).cuda())
  table = layer._table_on(torch.device("cuda", torch.cuda.current_device()))
  mapping = {int(v): i + 1 for i, v in enumerate(vocab.tolist())}
  res = {}
  for name, (pos, oov) in _batches(rng, V).items():
    x = np.where(oov, rng.randint(-2**62, 2**62, size=B, dtype=np.int64), vocab[pos])
    xd = torch.from_numpy(x).cuda()
    dev = _windows(lambda: ops.lookup(table, xd, 1, 1), args.windows, args.calls)
    host = _host(lambda: torch.from_numpy(np.asarray([mapping.get(v, 0) for v in x.tolist()], np.int64)).cuda(),
                 args.windows)
    assert torch.equal(layer(xd).cpu(), torch.from_numpy(np.asarray([mapping.get(v, 0) for v in x.tolist()])))
    res[name] = {"device_lookup": _summary(dev, B, B * 28), "host_dict_and_upload": _summary(host, B)}
  return res


def bench_str(V, args, rng):
  alphabet = "abcdefghijklmnopqrstuvwxyz ABCDEFGHIJKLMNOPQRSTUVWXYZ0123456789"
  lens = rng.randint(8, 65, size=V)
  vocab = np.array([f"{i:07d}:" + (alphabet * 2)[i % 60: i % 60 + n - 8] for i, n in enumerate(lens)])
  layer = StringLookup(vocabulary=vocab)
  dev0 = torch.device("cuda", torch.cuda.current_device())
  table = layer._table_on(dev0)
  mapping = {v: i + 1 for i, v in enumerate(vocab.tolist())}
  res = {}
  for name, (pos, oov) in _batches(rng, V).items():
    x = vocab[pos].astype(object)
    x[oov] = [s[:-1] + "#" for s in x[oov]]
    x = x.astype(vocab.dtype)
    data, offsets, _ = pack_strings(x)
    byts, offs = upload_packed(data, offsets, dev0)
    nbytes = B * (8 + 4 + 8 + 16 + 8) + 2 * int(offsets[-1])
    dev = _windows(lambda: ops.lookup(table, (byts, offs), 1, 1), args.windows, args.calls)
    pack = _host(lambda: pack_strings(x), args.windows)
    upload = _host(lambda: upload_packed(data, offsets, dev0), args.windows)
    call = _host(lambda: layer(x), args.windows)
    host = _host(lambda: torch.from_numpy(np.asarray([mapping.get(v, 0) for v in x.tolist()], np.int64)).cuda(),
                 args.windows)
    assert torch.equal(layer(x).cpu(), torch.from_numpy(np.asarray([mapping.get(v, 0) for v in x.tolist()])))
    res[name] = {"device_lookup": _summary(dev, B, nbytes), "host_pack_strings": _summary(pack, B),
                 "host_to_device_copy": _summary(upload, B), "layer_call_end_to_end": _summary(call, B),
                 "host_dict_and_upload": _summary(host, B), "mean_string_bytes": round(int(offsets[-1]) / B, 1)}
  return res


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--windows", type=int, default=7)
  ap.add_argument("--calls", type=int, default=50)
  ap.add_argument("--out", default=None)
  args = ap.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit("bench_lookup needs a CUDA device; no number is measured without one")
  rng = np.random.RandomState(0)
  out = {"card": _card(), "batch": B, "windows": args.windows, "calls_per_window": args.calls,
         "IntegerLookup_V1M": bench_int(1 << 20, args, rng), "IntegerLookup_V10M": bench_int(10 << 20, args, rng),
         "StringLookup_V1M": bench_str(1 << 20, args, rng)}
  text = json.dumps(out, indent=1)
  print(text)
  if args.out:
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as fh:
      fh.write(text)


if __name__ == "__main__":
  main()
