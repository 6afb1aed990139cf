"""Times K16 (TextVectorization) and K17 (Discretization, Normalization, masked GlobalAveragePooling1D) on the device,
against the host work they replace.

    python tools/bench_text.py [--windows 7] [--calls 50] [--out results.json]

Cases:
  - text: 4096 tutorial-like titles ("Word Word (1995)", 20-60 bytes) and 65536 strings of 40-200 bytes, with a 10 000
    token vocabulary.  Device time per call of the two K16 launches on already uploaded bytes, with
    output_sequence_length given (no host read): CUDA events around `calls` back-to-back calls, several windows, the
    median with the spread.  Host packing (pack_strings) and the one host-to-device copy, and a host tokenizer (`re`
    split of the lowercased, punctuation-stripped string, a dict per token, np.asarray, the upload), on the host clock.
  - numeric, B = 65536: bucketize of int64 timestamps over 1000 boundaries, normalize, and the masked mean pool forward
    and backward of [B, 20, 32] float32.
The card's name and power limit are read in the same run."""
from __future__ import annotations

import argparse
import json
import os
import re
import statistics
import string
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from recommenders_b200 import ops  # noqa: E402
from recommenders_b200._strings import pack_strings, upload_packed  # noqa: E402
from recommenders_b200.layers.preprocessing import TextVectorization  # noqa: E402

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


def _summary(per):
  return {"median_us": statistics.median(per), "min_us": min(per), "max_us": max(per)}


def _titles(rng, n, words):
  return np.array([" ".join(words[rng.randint(0, len(words), rng.randint(1, 6))]).title() + f" ({1920 + rng.randint(0, 80)})"
                   for _ in range(n)])


def _long(rng, n, words):
  seps = [" ", ", ", ". ", "! ", "\t"]
  out = []
  for _ in range(n):
    target = rng.randint(40, 201)
    idx, sep = rng.randint(0, len(words), 40), rng.randint(0, len(seps), 40)
    out.append("".join(words[i] + seps[j] for i, j in zip(idx, sep))[:target])
  return np.array(out)


def bench_text(windows, calls):
  rng = np.random.RandomState(0)
  words = np.array([f"Word{i}" for i in range(20_000)])
  vocab = [w.lower() for w in words[:10_000]]
  tv = TextVectorization(vocabulary=vocab, output_sequence_length=32)
  table = tv._lookup_layer._table_on(torch.device("cuda", torch.cuda.current_device()))
  strip = re.compile("[" + re.escape(string.punctuation) + "]")
  index = {w: i + 2 for i, w in enumerate(vocab)}
  out = {}
  for name, strings in (("titles_4096", _titles(rng, 4096, words)), ("strings_65536_40_200B", _long(rng, B, words))):
    data, offsets, _ = pack_strings(strings)
    byts, offs = upload_packed(data, offsets, torch.device("cuda"))
    dev = _windows(lambda: ops.text_vectorize(table, byts, offs, ops.TEXT_LOWER | ops.TEXT_STRIP, 32, 2, 1), windows,
                   calls)
    pack = _host(lambda: pack_strings(strings), windows)
    upload = _host(lambda: upload_packed(data, offsets, torch.device("cuda")), windows)
    layer = _host(lambda: tv(strings), windows)

    def host_tokenizer():
      rows = [[index.get(t, 1) for t in strip.sub("", s.lower()).split()][:32] for s in strings.tolist()]
      a = np.zeros((len(rows), 32), np.int64)
      for i, r in enumerate(rows):
        a[i, :len(r)] = r
      return torch.from_numpy(a).cuda()

    host = _host(host_tokenizer, windows, reps=1)
    assert torch.equal(host_tokenizer(), tv(strings))
    out[name] = {"n": len(strings), "bytes": int(data.size), "device_us": _summary(dev),
                 "host_pack_us": _summary(pack), "host_upload_us": _summary(upload),
                 "layer_call_us": _summary(layer), "host_re_dict_tokenizer_us": _summary(host)}
  return out


def bench_numeric(windows, calls):
  rng = np.random.RandomState(1)
  ts = torch.from_numpy(rng.randint(874724710, 893286638, size=B).astype(np.int64)).cuda()
  bounds = torch.from_numpy(np.linspace(874724710, 893286638, 1000).astype(np.float32)).cuda()
  mean, var = torch.tensor([8.8e8], device="cuda"), torch.tensor([2.9e13], device="cuda")
  x = torch.randn(B, 20, 32, device="cuda")
  ids = torch.from_numpy(rng.randint(0, 3, size=(B, 20))).cuda()
  g = torch.randn(B, 32, device="cuda")
  res = {
      "bucketize_int64_1000_bounds": _windows(lambda: ops.bucketize(ts, bounds), windows, calls),
      "normalize_int64": _windows(lambda: ops.normalize(ts, mean, var), windows, calls),
  }
  xg = x.clone().requires_grad_(True)

  def fwd():
    return ops.mean_pool(x, ids)

  def bwd():
    out = ops.mean_pool(xg, ids)
    torch.autograd.grad(out, xg, g)

  res["mean_pool_fwd_B65536_T20_d32"] = _windows(fwd, windows, calls)
  res["mean_pool_fwd_bwd_B65536_T20_d32"] = _windows(bwd, windows, calls)
  return {k: _summary(v) for k, v in res.items()}


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--windows", type=int, default=7)
  ap.add_argument("--calls", type=int, default=50)
  ap.add_argument("--out", default=None)
  a = ap.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit("bench_text.py needs a CUDA device")
  res = {"card": _card(), "text": bench_text(a.windows, a.calls), "numeric": bench_numeric(a.windows, a.calls)}
  s = json.dumps(res, indent=1)
  print(s)
  if a.out:
    with open(a.out, "w") as fh:
      fh.write(s)


if __name__ == "__main__":
  main()
