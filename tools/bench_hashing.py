"""Times K18, tf-keras `Hashing` on the device (ops.hashing / layers.Hashing).

    python tools/bench_hashing.py [--windows 7] [--calls 20] [--out results.json]

Cases:
  - ops.hashing on 2^22 int64 ids (uniform over int64), unsalted (FarmHash Fingerprint64) and salted (SipHash-2-4);
  - ops.hashing on 2^22 strings of title-like lengths, 10-90 bytes (uniform), already on the device, both hashes;
  - the uet tutorial's HashEmbeddingModel towers: five `Sequential([Hashing(b), Embedding(b, 32)])` over string features
    at batch 4096, next to the same five features through `Sequential([StringLookup(vocab), Embedding(V + 1, 32)])`.
    Device-only (inputs packed and uploaded once) and whole layer calls from NumPy strings (packing and upload included).
Device time per call: CUDA events around `calls` back-to-back calls after a warm-up, in several windows; the median
with the spread.  Values/s, and bytes read + written over kernel time: ints 8 (value) + 8 (bin); strings 8 (offset) +
len (bytes) + 8 (bin) -- every value's bytes read once.  The card's name and power limit are read in the same run."""
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
from recommenders_b200.layers.embedding import Embedding  # noqa: E402
from recommenders_b200.layers.preprocessing import Hashing, StringLookup  # noqa: E402

HBM_BYTES_PER_S = 3.35e12
N = 1 << 22
B = 4096
BUCKETS = {"movie_id": 600, "user_id": 400, "user_gender": 20, "user_zip_code": 400, "user_occupation_text": 20}


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


def _host(fn, windows, reps=5):
  fn()
  torch.cuda.synchronize()
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
         "values_per_s": n / (med * 1e-6)}
  if nbytes is not None:
    out["modelled_bytes"] = int(nbytes)
    out["bytes_per_s"] = nbytes / (med * 1e-6)
    out["share_of_3.35TB/s"] = round(nbytes / (med * 1e-6) / HBM_BYTES_PER_S, 4)
  return out


def bench_ints(args, rng):
  x = torch.from_numpy(rng.randint(-2**63, 2**63 - 1, size=N, dtype=np.int64)).cuda()
  res = {}
  for name, salt in (("unsalted_farmhash", None), ("salted_siphash", 133)):
    per = _windows(lambda: ops.hashing(x, 200_000, salt), args.windows, args.calls)
    res[name] = _summary(per, N, N * 16)
  return res


def bench_strings(args, rng):
  lens = rng.randint(10, 91, size=N)
  pool = rng.randint(32, 127, size=int(lens.sum()), dtype=np.uint8)
  offsets = np.zeros(N + 1, np.int64)
  np.cumsum(lens, out=offsets[1:])
  byts, offs = upload_packed(pool, offsets, torch.device("cuda", torch.cuda.current_device()))
  nbytes = N * 16 + int(offsets[-1])
  res = {"mean_string_bytes": round(float(lens.mean()), 1)}
  for name, salt in (("unsalted_farmhash", None), ("salted_siphash", 133)):
    per = _windows(lambda: ops.hashing((byts, offs), 200_000, salt), args.windows, args.calls)
    res[name] = _summary(per, N, nbytes)
  return res


def _features(rng):
  uid, mid = rng.randint(0, 943, size=B), rng.randint(0, 1682, size=B)
  occ = np.array(["doctor", "artist", "student", "other", "lawyer", "K-12 student", "retired", "writer", "engineer"])
  return {"movie_id": np.char.mod("%d", mid + 1), "user_id": np.char.mod("%d", uid + 1),
          "user_gender": np.where(uid % 2 == 0, "True", "False"), "user_zip_code": np.char.mod("%05d", uid * 37 % 100000),
          "user_occupation_text": occ[uid % len(occ)]}


def bench_towers(args, rng):
  feats = _features(rng)
  vocabs = {f: np.unique(v) for f, v in feats.items()}
  hash_towers = {f: torch.nn.Sequential(Hashing(num_bins=b), Embedding(b, 32)) for f, b in BUCKETS.items()}
  lookup_towers = {f: torch.nn.Sequential(StringLookup(vocabulary=vocabs[f], mask_token=None),
                                          Embedding(len(vocabs[f]) + 1, 32)) for f in BUCKETS}
  dev = torch.device("cuda", torch.cuda.current_device())
  packed = {}
  for f, v in feats.items():
    data, offsets, _ = pack_strings(v)
    packed[f] = upload_packed(data, offsets, dev)
  tables = {f: t[0]._table_on(dev) for f, t in lookup_towers.items()}

  def hash_device():
    return [hash_towers[f][1](ops.hashing(packed[f], b)) for f, b in BUCKETS.items()]

  def lookup_device():
    return [lookup_towers[f][1](ops.lookup(tables[f], packed[f], 1, 0)) for f in BUCKETS]

  def hash_layers():
    return [hash_towers[f](feats[f]) for f in BUCKETS]

  def lookup_layers():
    return [lookup_towers[f](feats[f]) for f in BUCKETS]

  res = {}
  with torch.no_grad():
    for name, fn in (("hashing_towers_device", hash_device), ("stringlookup_towers_device", lookup_device)):
      res[name] = _summary(_windows(fn, args.windows, args.calls), 5 * B)
    for name, fn in (("hashing_towers_layer_calls", hash_layers), ("stringlookup_towers_layer_calls", lookup_layers)):
      res[name] = _summary(_host(fn, args.windows), 5 * B)
  return res


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--windows", type=int, default=7)
  ap.add_argument("--calls", type=int, default=20)
  ap.add_argument("--out", default=None)
  args = ap.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit("bench_hashing needs a CUDA device; no number is measured without one")
  rng = np.random.RandomState(0)
  out = {"card": _card(), "windows": args.windows, "calls_per_window": args.calls,
         "int64_ids_2^22": bench_ints(args, rng), "strings_10_90_bytes_2^22": bench_strings(args, rng),
         "uet_towers_batch_4096": bench_towers(args, rng)}
  text = json.dumps(out, indent=1)
  print(text)
  if args.out:
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as fh:
      fh.write(text)


if __name__ == "__main__":
  main()
