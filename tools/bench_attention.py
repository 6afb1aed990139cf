"""Times K21 (the MultiHeadAttention core, ops.attention_core) and K22 (ops.layer_norm) on the device, next to torch's
scaled_dot_product_attention and layer_norm (fp32, TF32 off) on the same inputs and masks in the same run.

    python tools/bench_attention.py [--windows 5] [--calls 20] [--out profiles/h100_attention.json]

Attention shapes (B, T, H, dk, mask): the sequential retrieval tutorial's (1024, 10, 2, 16, causal), a SASRec tower's
(256, 200, 2, 32, causal) and a title encoder's (1024, 32, 4, 64, a padding mask on the keys); S = T, dv = dk.  Per
shape the forward (under no_grad) and the forward + backward (Q, K and V requiring gradients, backward from a fixed dO).
Ours reads Q, K, V as [B, T, H*dk] (the projections' layout); torch's SDPA gets [B, H, T, dk] copies made before the
timing.  LayerNorm at d = 32, 256 and 1024 over 65536 rows, forward and forward + backward (x, gamma, beta).
Device time per call: CUDA events around `calls` back-to-back calls after a warm-up, in several windows; the median with
the spread (bench_gru's helpers).  Outputs of both are compared.  The card's name and power limit are read in the same
run."""
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

SHAPES = [("tutorial", 1024, 10, 2, 16, "causal"), ("sasrec", 256, 200, 2, 32, "causal"),
          ("title_encoder", 1024, 32, 4, 64, "padding")]
LN_WIDTHS = [32, 256, 1024]
LN_ROWS = 65536


def bench_attention(name, B, T, H, d, mask, windows, calls):
  g = torch.Generator(device="cuda").manual_seed(B + T + H + d)
  Q, K, V, dO = (torch.randn((B, T, H * d), device="cuda", generator=g) for _ in range(4))
  causal = mask == "causal"
  vm = None
  if mask == "padding":
    lengths = torch.randint(1, T + 1, (B, 1), device="cuda", generator=g)
    vm = torch.arange(T, device="cuda")[None] < lengths
  heads = lambda t: t.reshape(B, T, H, d).transpose(1, 2).contiguous()
  q4, k4, v4, do4 = (heads(t) for t in (Q, K, V, dO))
  am = None if vm is None else vm[:, None, None, :]
  leaves = [t.clone().requires_grad_() for t in (Q, K, V)]
  tleaves = [t.clone().requires_grad_() for t in (q4, k4, v4)]

  def ours_fwd():
    with torch.no_grad():
      return ops.attention_core(Q, K, V, H, value_mask=vm, causal=causal)[0]

  def ours_step():
    for t in leaves:
      t.grad = None
    O, _ = ops.attention_core(*leaves, H, value_mask=vm, causal=causal)
    O.backward(dO)

  def torch_fwd():
    with torch.no_grad():
      return F.scaled_dot_product_attention(q4, k4, v4, attn_mask=am, is_causal=causal)

  def torch_step():
    for t in tleaves:
      t.grad = None
    F.scaled_dot_product_attention(*tleaves, attn_mask=am, is_causal=causal).backward(do4)

  diff = (ours_fwd().reshape(B, T, H, d).transpose(1, 2) - torch_fwd()).abs().max().item()
  row = {"shape": name, "B": B, "T": T, "S": T, "H": H, "dk": d, "dv": d, "mask": mask,
         "ours_fwd": _windows(ours_fwd, windows, calls), "torch_sdpa_fwd": _windows(torch_fwd, windows, calls),
         "ours_fwd_bwd": _windows(ours_step, windows, calls), "torch_sdpa_fwd_bwd": _windows(torch_step, windows, calls),
         "max_abs_diff_O_vs_sdpa": diff}
  row["fwd_speedup_vs_sdpa"] = round(row["torch_sdpa_fwd"]["us_median"] / row["ours_fwd"]["us_median"], 3)
  row["fwd_bwd_speedup_vs_sdpa"] = round(row["torch_sdpa_fwd_bwd"]["us_median"] / row["ours_fwd_bwd"]["us_median"], 3)
  return row


def bench_layer_norm(d, windows, calls):
  g = torch.Generator(device="cuda").manual_seed(d)
  x = torch.randn((LN_ROWS, d), device="cuda", generator=g)
  gamma, beta = torch.randn(d, device="cuda", generator=g), torch.randn(d, device="cuda", generator=g)
  dy = torch.randn((LN_ROWS, d), device="cuda", generator=g)
  leaves = [t.clone().requires_grad_() for t in (x, gamma, beta)]
  tleaves = [t.clone().requires_grad_() for t in (x, gamma, beta)]

  def ours_fwd():
    with torch.no_grad():
      return ops.layer_norm(x, gamma, beta, 1e-3)

  def ours_step():
    for t in leaves:
      t.grad = None
    ops.layer_norm(*leaves, 1e-3).backward(dy)

  def torch_fwd():
    with torch.no_grad():
      return F.layer_norm(x, (d,), gamma, beta, 1e-3)

  def torch_step():
    for t in tleaves:
      t.grad = None
    F.layer_norm(tleaves[0], (d,), tleaves[1], tleaves[2], 1e-3).backward(dy)

  row = {"rows": LN_ROWS, "d": d, "max_abs_diff_vs_torch": (ours_fwd() - torch_fwd()).abs().max().item(),
         "ours_fwd": _windows(ours_fwd, windows, calls), "torch_fwd": _windows(torch_fwd, windows, calls),
         "ours_fwd_bwd": _windows(ours_step, windows, calls), "torch_fwd_bwd": _windows(torch_step, windows, calls)}
  row["fwd_speedup_vs_torch"] = round(row["torch_fwd"]["us_median"] / row["ours_fwd"]["us_median"], 3)
  row["fwd_bwd_speedup_vs_torch"] = round(row["torch_fwd_bwd"]["us_median"] / row["ours_fwd_bwd"]["us_median"], 3)
  return row


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--windows", type=int, default=5)
  ap.add_argument("--calls", type=int, default=20)
  ap.add_argument("--out", default=None)
  args = ap.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit("bench_attention needs a CUDA device; no number is measured without one")
  torch.backends.cuda.matmul.allow_tf32 = False
  torch.backends.cudnn.allow_tf32 = False
  out = {"card": _card(), "windows": args.windows, "calls_per_window": args.calls,
         "attention": [bench_attention(*s, args.windows, args.calls) for s in SHAPES],
         "layer_norm": [bench_layer_norm(d, args.windows, args.calls) for d in LN_WIDTHS]}
  text = json.dumps(out, indent=1)
  print(text)
  if args.out:
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as fh:
      fh.write(text + "\n")


if __name__ == "__main__":
  main()
