"""Debug driver for the tensor-core top-K path: compares tfrs_topk_tc_f32 with the exact CUDA-core
scan on one shape and prints mismatch statistics.  usage: python tools/tc_check.py Q N d k [seed]"""
import sys, time
import os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from recommenders_b200 import ops

Q, N, d, k = [int(x) for x in sys.argv[1:5]]
seed = int(sys.argv[5]) if len(sys.argv) > 5 else 0
dev = torch.device("cuda", 0)
g = torch.Generator(device=dev); g.manual_seed(seed)
c = torch.randn((N, d), generator=g, device=dev); q = torch.randn((Q, d), generator=g, device=dev)
print("tc_supported:", ops.tc_supported(Q, N, d, k), flush=True)
t0 = time.time(); idx = ops.index_build(c); torch.cuda.synchronize(); print("index_build ok %.3fs" % (time.time() - t0), flush=True)
s, i = ops.topk_tc(q, c, idx, k); torch.cuda.synchronize(); print("topk_tc ok", flush=True)
print("stats:", ops.tc_last_call_stats(Q, N, d, k))
Qc = min(Q, 128)
es, ei = ops.topk_scan(q[:Qc], c, k); torch.cuda.synchronize()
print("stats:", ops.tc_last_call_stats(Q, N, d, k))
print("ids equal:", bool((i[:Qc] == ei).all()), " scores equal:", bool((s[:Qc] == es).all()))
if not (i[:Qc] == ei).all():
  bad = (i[:Qc] != ei).any(1).nonzero().flatten()
  print("bad rows:", bad.numel(), bad[:10].tolist())
  r = int(bad[0]); print(i[r][:12].tolist()); print(ei[r][:12].tolist()); print(s[r][:6].tolist()); print(es[r][:6].tolist())
ops.profile_enable(True)
for _ in range(5): ops.topk_tc(q, c, idx, k)
ms, calls = ops.profile_read(); ops.profile_enable(False)
print("stage ms/call (prep, sample, filter, finalize):", [round(m / calls, 4) for m in ms], "total %.4f" % (sum(ms) / calls))
print("filter TFLOP/s: %.1f   q/s: %.0f" % (2.0 * Q * N * d / (ms[2] / calls * 1e-3) / 1e12, Q / (sum(ms) / calls * 1e-3)))

if os.environ.get("TC_DEBUG"):
  import ctypes
  from recommenders_b200 import _ffi
  out = (ctypes.c_int64 * 10)(); _ffi.lib().tfrs_topk_tc_layout(Q, N, d, k, out)
  o_count, o_ovf, o_thr, o_cand, parts, cap, Qp, o_cut = [int(x) for x in out[:8]]
  ws = _ffi.workspace(0, dev, "tc"); base = (-ws.data_ptr()) % 16
  thr = ws[base + o_thr: base + o_thr + Q * 4].view(torch.float32)
  cut = ws[base + o_cut: base + o_cut + Q * 4].view(torch.float32)
  hdr = idx[:64].view(torch.int32)
  print("hdr ints:", hdr[:12].tolist(), "max_norm2", idx[:4].view(torch.float32).item(), "amax", idx[4:8].view(torch.float32).item())
  ec = int(hdr[2])
  amax_q = float(q.abs().max()); import math
  eq = 15 - math.frexp(amax_q)[1]
  S = (torch.ldexp(q[:8], torch.tensor(eq, device=dev)).half().float() @ torch.ldexp(c, torch.tensor(ec, device=dev)).half().float().T)
  kth = S.topk(k, dim=1).values[:, -1]
  print("eq", eq, "ec", ec)
  print("thr[:8]   ", thr[:8].tolist())
  print("kth[:8]   ", kth.tolist())
  print("max[:8]   ", S.max(1).values.tolist())
  print("cut[:8]   ", cut[:8].tolist())
  # decode a few elements of the corpus image and of the query image
  img = idx[1024:]
  def elem(buf, row, kk, kb=1):
    t, r = divmod(row, 128); slab, kq = divmod(kk, 64); cj, w = divmod(kq, 8)
    off = t * kb * 16384 + slab * 16384 + r * 128 + ((cj ^ (r & 7)) * 16) + w * 2
    return buf[off:off + 2].view(torch.float16).item()
  for (row, kk) in [(0, 0), (5, 3), (130, 17), (199999, 63)]:
    print("corpus img", row, kk, elem(img, row, kk, (d + 63) // 64), "expected", float(torch.ldexp(c[row, kk], torch.tensor(ec, device=dev)).half()))
  qst = ws[base: base + 16].view(torch.int32)
  print("qst:", qst.tolist(), "amax_q", ws[base + 4: base + 8].view(torch.float32).item())
  qimg = ws[base + 1024:]
  for (row, kk) in [(0, 0), (5, 3), (130, 17)]:
    print("query img", row, kk, elem(qimg, row, kk, (d + 63) // 64), "expected", float(torch.ldexp(q[row, kk], torch.tensor(int(qst[2]), device=dev)).half()))
