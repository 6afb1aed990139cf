"""Times the dense attention layers' core (ops.dense_attention: K21's dot scores, K25's concat and additive scores) on the
device, next to a plain torch formulation (fp32, TF32 off) on the same inputs and masks in the same run.

    python tools/bench_dense_attention.py [--windows 5] [--calls 20] [--out profiles/h100_dense_attention.json]

Shapes (B, Tq, Tv, d, mask): DIN-style target attention, one candidate over a padded history, (4096, 1, 50 or 200, 32
or 64, a padding mask on the values); BST-style self attention (1024, 20, 20, 64, causal).  dv = d.  Each shape in the
dot, concat and additive modes with a scale, at dropout 0 and 0.1 (training).  Per case the forward (under no_grad)
and the forward + backward (query, key, value and the weights requiring gradients, backward from a fixed dO).  The
torch formulation is what a user would write: q @ k^T (dot) or the [B, Tq, Tv, d] tanh tensor (concat, additive), the
-1e9 mask, softmax, torch's dropout, @ v.  Device time per call: CUDA events around `calls` back-to-back calls after a
warm-up, in several windows; the median with the spread (bench_gru's helpers).  At dropout 0 the outputs of both are
compared.  The card's name and power limit are read in the same run."""
from __future__ import annotations

import argparse
import json
import os
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from bench_gru import _card, _windows  # noqa: E402
from recommenders_b200 import ops  # noqa: E402

SHAPES = [("din", 4096, 1, 50, 32, "padding"), ("din", 4096, 1, 50, 64, "padding"),
          ("din", 4096, 1, 200, 32, "padding"), ("din", 4096, 1, 200, 64, "padding"),
          ("bst", 1024, 20, 20, 64, "causal")]
MODES = ("dot", "concat", "additive")
RATES = (0.0, 0.1)


def _torch_core(q, k, v, mode, scale, cw, vm, causal, rate):
  if mode == "dot":
    s = (q @ k.transpose(1, 2)) * scale
  else:
    u = q[:, :, None, :] + k[:, None, :, :]
    s = cw * torch.tanh(scale * u).sum(-1) if mode == "concat" else (torch.tanh(u) * scale).sum(-1)
  keep = torch.ones(s.shape, dtype=torch.bool, device=s.device)
  if vm is not None:
    keep = keep & vm[:, None, :]
  if causal:
    keep = keep & torch.ones(s.shape[1:], dtype=torch.bool, device=s.device).tril()[None]
  w = torch.softmax(s - 1e9 * (~keep).float(), -1)
  if rate:
    w = F.dropout(w, rate, training=True)
  return w @ v


def bench_case(name, B, Tq, Tv, d, mask, mode, rate, windows, calls):
  g = torch.Generator(device="cuda").manual_seed(B + Tq + Tv + d)
  q = torch.randn((B, Tq, d), device="cuda", generator=g)
  k, v = (torch.randn((B, Tv, d), device="cuda", generator=g) for _ in range(2))
  dO = torch.randn((B, Tq, d), device="cuda", generator=g)
  scale = torch.rand((d,) if mode == "additive" else (), device="cuda", generator=g) + 0.5
  cw = torch.ones((), device="cuda") if mode == "concat" else None
  causal = mask == "causal"
  vm = None
  if mask == "padding":
    lengths = torch.randint(1, Tv + 1, (B, 1), device="cuda", generator=g)
    vm = torch.arange(Tv, device="cuda")[None] < lengths
  leaves = [t.clone().requires_grad_() for t in (q, k, v, scale)] + ([cw.clone().requires_grad_()] if cw is not None
                                                                     else [None])
  tleaves = [None if t is None else t.clone().requires_grad_() for t in leaves]
  calls_made = [0]

  def ours(*t):
    calls_made[0] += 1
    return ops.dense_attention(t[0], t[1], t[2], mode, t[3], t[4], value_mask=vm, causal=causal, rate=rate, seed=7,
                               call=calls_made[0])[0]

  def ours_fwd():
    with torch.no_grad():
      return ours(q, k, v, scale, cw)

  def ours_step():
    for t in leaves:
      if t is not None:
        t.grad = None
    ours(*leaves).backward(dO)

  def torch_fwd():
    with torch.no_grad():
      return _torch_core(q, k, v, mode, scale, cw, vm, causal, rate)

  def torch_step():
    for t in tleaves:
      if t is not None:
        t.grad = None
    _torch_core(*tleaves[:3], mode, tleaves[3], tleaves[4], vm, causal, rate).backward(dO)

  row = {"shape": name, "B": B, "Tq": Tq, "Tv": Tv, "d": d, "mask": mask, "mode": mode, "dropout": rate,
         "ours_fwd": _windows(ours_fwd, windows, calls), "torch_fwd": _windows(torch_fwd, windows, calls),
         "ours_fwd_bwd": _windows(ours_step, windows, calls), "torch_fwd_bwd": _windows(torch_step, windows, calls)}
  if not rate:
    row["max_abs_diff_vs_torch"] = (ours_fwd() - torch_fwd()).abs().max().item()
  row["fwd_speedup_vs_torch"] = round(row["torch_fwd"]["us_median"] / row["ours_fwd"]["us_median"], 3)
  row["fwd_bwd_speedup_vs_torch"] = round(row["torch_fwd_bwd"]["us_median"] / row["ours_fwd_bwd"]["us_median"], 3)
  print(json.dumps({k: row[k] for k in ("shape", "Tv", "d", "mode", "dropout", "fwd_speedup_vs_torch",
                                        "fwd_bwd_speedup_vs_torch")}), flush=True)
  return row


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--windows", type=int, default=5)
  ap.add_argument("--calls", type=int, default=20)
  ap.add_argument("--out", default=None)
  args = ap.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit("bench_dense_attention needs a CUDA device; no number is measured without one")
  torch.backends.cuda.matmul.allow_tf32 = False
  torch.backends.cudnn.allow_tf32 = False
  out = {"card": _card(), "windows": args.windows, "calls_per_window": args.calls,
         "dense_attention": [bench_case(*s, m, r, args.windows, args.calls) for s in SHAPES for m in MODES
                             for r in RATES]}
  text = json.dumps(out, indent=1)
  if args.out:
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as fh:
      fh.write(text + "\n")


if __name__ == "__main__":
  main()
