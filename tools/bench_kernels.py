"""Secondary measurements for BASELINE.md §4 (configs 3 and 5): embedding gather GB/s, sparse Adagrad,
in-batch softmax step, Cross layer, ClippyAdagrad.  CUDA events, warm-up, inputs larger than L2 or rotated between
iterations.  Prints one JSON object.
usage: python tools/bench_kernels.py [--quick] [--top-stack-only | --optimizers-only | --unified-only]"""
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from recommenders_b200 import ops

dev = torch.device("cuda", 0)
quick = "--quick" in sys.argv
peaks = {}
try:
  peaks = json.load(open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "MEASURED_PEAKS.json")))
except Exception:
  pass
HBM = peaks.get("hbm_gbs", 3350.0)   # H100 SXM data sheet when not measured


def timeit(fn, iters=20, warm=5):
  for _ in range(warm):
    fn()
  torch.cuda.synchronize()
  e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  e0.record()
  for _ in range(iters):
    fn()
  e1.record()
  torch.cuda.synchronize()
  return e0.elapsed_time(e1) / iters * 1e-3


def graph_time(fn, iters=20):
  """One call captured in a CUDA graph and replayed: device time.  (The Python binding of a 26-table gather costs more host
  time than the kernel runs, so a plain Python loop measures the host, with run-to-run differences of 25 %.)"""
  fn(); torch.cuda.synchronize()
  gr = torch.cuda.CUDAGraph()
  with torch.cuda.graph(gr):
    fn()
  return timeit(gr.replay, iters=iters)


out = {"hbm_peak_gbs": HBM}
g = torch.Generator(device=dev); g.manual_seed(7)


def unified_legs():
  """K8 (UnifiedEmbedding) at the cfg5 shape: 26 int64 features x 2 chunks over UnifiedEmbeddingConfig(13M buckets,
  dim 16, 4 tables) -- cfg5's parameter count (26 x 1M x 32) and its [65536, 832] activation.  Ids uniform in [0, 1M)
  and Zipf(1.05).  Device times are CUDA-graph replays.  Algorithmic bytes of the forward: the 52 rows read and the
  activation written, the ids read and the bucket ids written (the training forward); the hash-only and K1-gather legs
  split that time into its hashing and its row traffic."""
  import subprocess
  import numpy as np
  from recommenders_b200.layers.feature_multiplexing import UnifiedEmbedding, UnifiedEmbeddingConfig
  B, F, V = (65536, 26, 1_000_000) if not quick else (8192, 26, 100_000)
  buckets, dim = (13_000_000 if not quick else 1_000_000), 16
  cfg = UnifiedEmbeddingConfig(buckets, dim, 4, "cfg5")
  for k in range(F):
    cfg.add_feature(f"f{k}", 2)
  layer = UnifiedEmbedding(cfg)
  rng = np.random.RandomState(7)
  g7 = torch.Generator(device=dev); g7.manual_seed(7)
  dists = {"uniform": [torch.randint(0, V, (B,), generator=g7, device=dev) for _ in range(F)],
           "zipf": [torch.from_numpy(np.minimum(rng.zipf(1.05, size=B) - 1, V - 1)).to(dev) for _ in range(F)]}
  width = 2 * F * dim
  act = torch.empty((B, width), device=dev)
  tables = [t.weight for t in layer._tables]
  chunks = [(k, t, key, pos) for k, (_, ch) in enumerate(layer._plan) for t, key, pos in ch]
  res = {}
  for kind, ids in dists.items():
    inputs = [ops.LookupInput(x) for x in ids]
    bins = [torch.empty(B, dtype=torch.int64, device=dev) for _ in chunks]
    slots = [ops.LookupSlot(k, tables[t], key, act, pos * dim, b) for (k, t, key, pos), b in zip(chunks, bins)]
    slots_inf = [s._replace(ids=None) for s in slots]
    t_fwd = graph_time(lambda: ops.unified_lookup(inputs, slots))
    t_inf = graph_time(lambda: ops.unified_lookup(inputs, slots_inf))
    t_hash = graph_time(lambda: [ops.hash_bins(ids[k], buckets, key) for k, _, key, _ in chunks])
    t_gather = graph_time(lambda: ops.gather([tables[t] for _, t, _, _ in chunks], bins, out=act,
                                             col_offsets=[pos * dim for _, _, _, pos in chunks]))
    grads = [torch.randn((B, width), generator=g7, device=dev)] * len(slots)
    rows = [torch.empty((B, dim), device=dev) for _ in slots]
    t_bwd = graph_time(lambda: ops.unified_lookup_bwd(inputs, slots, grads, rows))
    n_slots = len(chunks)
    by_fwd = B * n_slots * dim * 4 + B * width * 4 + B * F * 8 + B * n_slots * 8
    by_gather = B * n_slots * dim * 4 + B * width * 4 + B * n_slots * 8
    by_bwd = B * width * 4 + B * n_slots * dim * 4
    res[kind] = {"fwd_seconds": t_fwd, "fwd_algorithmic_bytes": by_fwd, "fwd_GBps": by_fwd / t_fwd / 1e9,
                 "fwd_frac_of_hbm": by_fwd / t_fwd / 1e9 / HBM, "fwd_no_bucket_ids_seconds": t_inf,
                 "hash_only_seconds": t_hash, "k1_gather_same_rows_seconds": t_gather,
                 "k1_gather_GBps": by_gather / t_gather / 1e9, "fwd_over_k1_gather": t_fwd / t_gather,
                 "bwd_seconds": t_bwd, "bwd_GBps": by_bwd / t_bwd / 1e9}
  # 26 string features end to end through the layer, host packing and the one upload included: host-bound
  words = {f"f{k}": np.char.mod("%d", dists["uniform"][k].cpu().numpy()) for k in range(F)}
  with torch.no_grad():
    res["strings_end_to_end_seconds"] = timeit(lambda: layer(words), iters=5, warm=2)
  try:
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True, timeout=30).stdout.strip().splitlines()[0]
  except Exception as e:  # the card name from torch is still reported
    smi = repr(e)
  res["device"] = torch.cuda.get_device_name(dev)
  res["nvidia_smi_name_power_limit"] = smi
  res["shape"] = f"{F} int64 features x 2 chunks, 4 tables {buckets}x{dim}, batch {B}"
  out["cfg5_unified_embedding"] = res


if "--unified-only" in sys.argv:
  unified_legs()
  print(json.dumps(out))
  sys.exit(0)


def optimizer_legs():
  """Sparse Adagrad (K4) and sparse ClippyAdagrad (K7) on the same B = 16384 batches of a 1M x 64 user table, uniform and
  Zipf(1.05) ids, then the dense ClippyAdagrad multi-tensor step of the cfg5 top stack.  Algorithmic bytes from the
  unique rows u of each batch: Adagrad n*d*4 + 4*u*d*4; ClippyAdagrad pass A n*d*4 + 3*u*d*4, pass B 5*u*d*4."""
  import numpy as np
  V, d, n = (1_000_000, 64, 16384) if not quick else (100_000, 64, 4096)
  table = (torch.rand((V, d), generator=g, device=dev) - 0.5) * 0.1
  acc_ag = torch.full_like(table, 0.1); acc_cl = torch.full_like(table, 0.1)
  grads = torch.randn((n, d), generator=g, device=dev) * 0.01
  rng = np.random.RandomState(3)
  batches = {"uniform": [torch.randint(0, V, (n,), generator=g, device=dev) for _ in range(4)],
             "zipf": [torch.from_numpy(np.minimum(rng.zipf(1.05, size=n) - 1, V - 1)).to(dev) for _ in range(4)]}
  res = {}
  for kind, ids in batches.items():
    u = sum(int(torch.unique(i).numel()) for i in ids) / len(ids)
    it = {"i": 0}

    def nxt():
      k = it["i"] % 4; it["i"] += 1
      return ids[k]
    t_ag = timeit(lambda: ops.sparse_adagrad_(table, acc_ag, nxt(), grads, 0.5), iters=50, warm=5)
    t_cl = timeit(lambda: ops.sparse_clippy_adagrad_(table, acc_cl, nxt(), grads, 0.5, 1e-7, 0.1, 1e-3, 1e-7), iters=50, warm=5)
    b_ag = n * d * 4 + 4 * u * d * 4
    b_cl = n * d * 4 + 8 * u * d * 4
    res[kind] = {"unique_rows": u, "adagrad_seconds": t_ag, "adagrad_GBps_algorithmic": b_ag / t_ag / 1e9,
                 "clippy_seconds": t_cl, "clippy_GBps_algorithmic": b_cl / t_cl / 1e9, "clippy_over_adagrad": t_cl / t_ag}
  res["shape"] = f"table {V}x{d}, batch {n}, ids int64, 4 batches rotated"
  out["cfg3_sparse_clippy_adagrad"] = res
  del table, acc_ag, acc_cl, grads, batches
  shapes = [(845, 512), (512,), (512, 256), (256,), (256, 1), (1,)]
  vs = [torch.randn(s, generator=g, device=dev) * 0.05 for s in shapes]
  gs = [torch.randn(s, generator=g, device=dev) * 0.01 for s in shapes]
  accs = [torch.full(s, 0.1, device=dev) for s in shapes]
  f = torch.zeros((len(shapes),), device=dev)
  t = timeit(lambda: ops.clippy_adagrad_dense_(vs, gs, accs, 0.05, 1e-7, 0.1, 1e-3, 1e-7, clipping_factors=f), iters=100, warm=10)
  N = sum(v.numel() for v in vs)
  out["cfg5_top_stack_clippy_dense_step"] = {"seconds": t, "elements": N, "variables": len(shapes),
                                             "GBps_algorithmic": 8 * N * 4 / t / 1e9, "launches": 3,
                                             "note": "init + pass A + pass B; bytes 3N*4 read (A) + 3N*4 read, 2N*4 written (B)"}


if "--optimizers-only" in sys.argv:
  optimizer_legs()
  print(json.dumps(out))
  sys.exit(0)

# ---- config 5 top stack (K6): MLP 845 -> 512 (relu) -> 256 (relu) -> 1 (sigmoid) at B = 65536, forward and forward + backward
#      (dx of the stack input, dW, db of every layer).  `--top-stack-only` prints this leg alone.
Bm, dims = (65536, [845, 512, 256, 1]) if not quick else (8192, [845, 512, 256, 1])
xm = torch.rand((Bm, dims[0]), generator=g, device=dev)
Wm = [(torch.randn((dims[i], dims[i + 1]), generator=g, device=dev) / dims[i] ** 0.5).requires_grad_(True) for i in range(3)]
bm = [torch.zeros((dims[i + 1],), device=dev, requires_grad=True) for i in range(3)]
gm = torch.randn((Bm, 1), generator=g, device=dev)
acts = ["relu", "relu", "sigmoid"]


def top_stack(x):
  for W, b, a in zip(Wm, bm, acts):
    x = ops.dense(x, W, b, a)
  return x


def top_stack_fb():
  x = xm.detach().requires_grad_(True)
  top_stack(x).backward(gm)


with torch.no_grad():
  t_f = timeit(lambda: top_stack(xm), iters=10 if not quick else 3, warm=3)
t_fb = timeit(top_stack_fb, iters=10 if not quick else 3, warm=3)
fl_f = sum(2.0 * Bm * dims[i] * dims[i + 1] for i in range(3))
PEAK_FP16 = peaks.get("bf16_tflops", 989.0)   # H100 SXM data sheet dense FP16 when not measured
out["cfg5_top_stack"] = {"fwd_seconds": t_f, "fwd_bwd_seconds": t_fb, "fwd_flops": fl_f, "fwd_bwd_flops": 3 * fl_f,
                         "fwd_TFLOPs": fl_f / t_f / 1e12, "fwd_bwd_TFLOPs": 3 * fl_f / t_fb / 1e12,
                         "fwd_bwd_frac_of_fp16_peak": 3 * fl_f / t_fb / 1e12 / PEAK_FP16, "peak_tflops": PEAK_FP16,
                         "shape": f"B={Bm}, {'->'.join(map(str, dims))}",
                         "path": "wgmma split-fp16 GEMMs (each product executed 3x) for the 512 / 256 layers, exact warp-per-row "
                                 "kernel for the 1-unit layer; algorithmic flops"}
del xm, Wm, bm, gm
if "--top-stack-only" in sys.argv:
  print(json.dumps(out))
  sys.exit(0)

# ---- config 5 gather: 26 tables 1M x 32, 65536 ids each -> [65536, 26*32 (+13 dense, ld 848)]
F, V, D, B = (26, 1_000_000, 32, 65536) if not quick else (26, 100_000, 32, 8192)
tables = [torch.rand((V, D), generator=g, device=dev) - 0.5 for _ in range(F)]
ids_sets = [[torch.randint(0, V, (B,), generator=g, device=dev, dtype=torch.int32) for _ in range(F)] for _ in range(4)]
act = torch.zeros((B, 848), device=dev)
state = {"i": 0}


def gather5():
  ops.gather(tables, ids_sets[state["i"] % 4], out=act); state["i"] += 1


t = sum(graph_time(lambda ids=ids: ops.gather(tables, ids, out=act)) for ids in ids_sets) / len(ids_sets)
t_host = timeit(gather5)
bytes5 = B * F * D * 4 * 2 + B * F * 4
out["cfg5_gather"] = {"seconds": t, "algorithmic_bytes": bytes5, "GBps": bytes5 / t / 1e9, "frac_of_hbm": bytes5 / t / 1e9 / HBM,
                      "python_loop_seconds": t_host, "timing": "CUDA-graph replays (device time); python_loop_seconds is host-bound",
                      "shape": f"{F} tables {V}x{D}, batch {B}, ids int32"}

# ---- config 5 Cross: B=65536, D=845 (ld 848 padded activations -> use D=848 contiguous here), 3 layers fwd
Dc = 845
x0 = torch.rand((B, Dc), generator=g, device=dev)
Ws = [torch.randn((Dc, Dc), generator=g, device=dev) * 0.05 for _ in range(3)]
bs = [torch.zeros((Dc,), device=dev) for _ in range(3)]


def cross3():
  x = x0
  for W, b in zip(Ws, bs):
    x = ops.cross(x0, x, W, b, 0.0)
  return x


with torch.no_grad():
  t = timeit(cross3, iters=5 if not quick else 3, warm=2)
flops = 3 * 2.0 * B * Dc * Dc
out["cfg5_cross_fwd_3layers"] = {"seconds": t, "TFLOPs": flops / t / 1e12, "flops": flops, "path": "wgmma fp16 hi/lo split GEMM + fused epilogue (B>=1024), exact CUDA-core SGEMM otherwise"}
# one Cross layer forward + backward (the training step's share), then the low-rank variants (p = 256) -- SURVEY 8f-4
go = torch.randn((B, Dc), generator=g, device=dev)
def cross_fb():
  xs = [t.detach().requires_grad_(True) for t in (x0, x0, Ws[0], bs[0])]
  ops.cross(xs[0], xs[1], xs[2], xs[3], 0.0).backward(go)
t = timeit(cross_fb, iters=5 if not quick else 3, warm=2)
out["cfg5_cross_layer_fwd_bwd"] = {"seconds": t, "TFLOPs": 3 * 2.0 * B * Dc * Dc / t / 1e12, "note": "fwd + dx + dW GEMMs, algorithmic flops"}
P = 256
Us = [torch.randn((Dc, P), generator=g, device=dev) * 0.05 for _ in range(3)]
Vs = [torch.randn((P, Dc), generator=g, device=dev) * 0.05 for _ in range(3)]
def lowrank3():
  x = x0
  for U, V, b in zip(Us, Vs, bs):
    x = ops.cross_lowrank(x0, x, U, V, b, 0.0)
  return x
def lowrank3_unfused():
  x = x0
  for U, V, b in zip(Us, Vs, bs):
    x = x0 * (ops.matmul(ops.matmul(x, U), V) + b) + x
  return x
with torch.no_grad():
  t = timeit(lowrank3, iters=5 if not quick else 3, warm=2)
  t0 = timeit(lowrank3_unfused, iters=3, warm=1)
fl = 3 * 2 * 2.0 * B * Dc * P
out["cfg5_multilayer_dcn_p256_fwd_3layers"] = {"seconds": t, "TFLOPs": fl / t / 1e12, "flops": fl, "unfused_cuda_core_seconds": t0,
                                               "path": "2 wgmma split-fp16 GEMMs per layer, cross formula in the second one's epilogue"}
def lowrank_fb():
  ys = [t.detach().requires_grad_(True) for t in (x0, x0, Us[0], Vs[0], bs[0])]
  ops.cross_lowrank(ys[0], ys[1], ys[2], ys[3], ys[4], 0.0).backward(go)
t = timeit(lowrank_fb, iters=5 if not quick else 3, warm=2)
out["cfg5_lowrank_layer_fwd_bwd"] = {"seconds": t, "TFLOPs": 3 * 2 * 2.0 * B * Dc * P / t / 1e12, "note": "2 fwd + 4 bwd GEMMs, algorithmic flops"}
del tables, ids_sets, act, x0, Ws, Us, Vs, go

# ---- config 3: two-tower step pieces, 10M users / 1M items, d=64, batch 16384
U, I, d, Bt = (10_000_000, 1_000_000, 64, 16384) if not quick else (1_000_000, 100_000, 64, 4096)
ut = (torch.rand((U, d), generator=g, device=dev) - 0.5) * 0.1
it = (torch.rand((I, d), generator=g, device=dev) - 0.5) * 0.1
uacc = torch.full_like(ut, 0.1); iacc = torch.full_like(it, 0.1)
uid = [torch.randint(0, U, (Bt,), generator=g, device=dev) for _ in range(4)]
iid = [torch.randint(0, I, (Bt,), generator=g, device=dev) for _ in range(4)]
state["i"] = 0


def gather3():
  k = state["i"] % 4; state["i"] += 1
  return ops.gather([ut], [uid[k]]), ops.gather([it], [iid[k]])


t = timeit(gather3)
bytes3 = 2 * Bt * d * 4 * 2 + 2 * Bt * 8
out["cfg3_gather_2tables"] = {"seconds": t, "algorithmic_bytes": bytes3, "GBps": bytes3 / t / 1e9, "frac_of_hbm": bytes3 / t / 1e9 / HBM,
                              "note": "2 launches of 4 MB each: launch-latency bound at this size"}
qe, ce = gather3()
qe = qe.requires_grad_(True); ce = ce.requires_grad_(True)


def softmax_fwd_bwd():
  qe.grad = None; ce.grad = None
  loss = ops.inbatch_softmax_loss(qe, ce)
  loss.backward()
  return loss


t = timeit(softmax_fwd_bwd, iters=5 if not quick else 3, warm=2)
out["cfg3_inbatch_softmax_fwd_bwd"] = {"seconds": t, "TFLOPs": 8.0 * Bt * Bt * d / t / 1e12, "flops": 8.0 * Bt * Bt * d,
                                       "path": "wgmma split-fp16 forward (online log-sum-exp) + wgmma backward (G as the register A operand)"}
with torch.no_grad():
  t = timeit(lambda: ops.inbatch_softmax_tc(qe, ce), iters=10, warm=3)
  out["cfg3_inbatch_softmax_fwd_only"] = {"seconds": t, "TFLOPs": 2.0 * Bt * Bt * d / t / 1e12}
  _, lse_t = ops.inbatch_softmax_tc(qe, ce)
  t = timeit(lambda: ops.inbatch_softmax_tc_bwd(qe, ce, lse_t), iters=10, warm=3)
  out["cfg3_inbatch_softmax_bwd_only"] = {"seconds": t, "TFLOPs": 4.0 * Bt * Bt * d / t / 1e12,
                                          "note": "algorithmic flops (dq + dc); the kernels also recompute S twice"}
gq = qe.grad.detach().clone()


def adagrad3():
  k = state["i"] % 4; state["i"] += 1
  ops.sparse_adagrad_(ut, uacc, uid[k], gq, 0.5)


t = timeit(adagrad3)
out["cfg3_sparse_adagrad_user_table"] = {"seconds": t, "rows": Bt, "GBps_algorithmic": (Bt * d * 4 * 5) / t / 1e9}
del ut, it, uacc, iacc
torch.cuda.empty_cache()
optimizer_legs()
# ---- Streaming over a corpus that lives in HOST memory (SURVEY 8f-1): 1M x 64 rows in pinned memory, dataset batches of
#      8192 rows coalesced into 262144-row chunks, pinned double-buffered H2D overlapped with the tensor-core scan per chunk
try:
  import recommenders_b200 as tfrs
  Ns, Qs, ks = (1_000_000, 4096, 100) if not quick else (200_000, 1024, 100)
  corpus_host = torch.randn((Ns, 64), generator=torch.Generator().manual_seed(1)).pin_memory()
  qd = torch.randn((Qs, 64), generator=g, device=dev)
  layer = tfrs.layers.factorized_top_k.Streaming(k=ks).index_from_dataset(
      tfrs.data.Dataset.from_tensor_slices(corpus_host).batch(8192))
  t = timeit(lambda: layer(qd), iters=3, warm=1)
  on_dev = tfrs.layers.factorized_top_k.Streaming(k=ks).index_from_dataset(
      tfrs.data.Dataset.from_tensor_slices(corpus_host.to(dev)).batch(8192))
  t_dev = timeit(lambda: on_dev(qd), iters=3, warm=1)
  out["streaming_host_corpus"] = {"seconds": t, "queries_per_s": Qs / t, "h2d_bytes": Ns * 64 * 4, "h2d_GBps": Ns * 64 * 4 / t / 1e9,
                                  "device_resident_seconds": t_dev, "device_resident_queries_per_s": Qs / t_dev,
                                  "shape": f"{Qs} queries x {Ns}x64 corpus in pinned host memory, top-{ks}"}
except Exception as e:  # keep the other figures if this leg fails
  out["streaming_host_corpus"] = {"error": repr(e)}
print(json.dumps(out))
