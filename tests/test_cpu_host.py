"""CPU-side tests (run with -m "not gpu"): the C-ABI library loads and exports every symbol that
include/tfrs_b200.h declares, the host logic (dataset shim, metric accumulators, in_top_k, error
behaviour without a GPU), and the sharded top-K protocol over gloo with world_size 2."""
import ctypes
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared_symbols():
  src = open(os.path.join(ROOT, "include", "tfrs_b200.h")).read()
  src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
  return sorted(set(re.findall(r"\b(tfrs_[a-z0-9_]+)\s*\(", src)))


def test_library_builds_and_exports_exactly_the_declared_symbols():
  from recommenders_b200 import build, _ffi
  path = build.build()
  assert os.path.exists(path)
  lib = ctypes.CDLL(path)
  declared = _declared_symbols()
  assert len(declared) >= 20
  for name in declared:
    assert hasattr(lib, name), f"{name} declared in include/tfrs_b200.h but not exported"
  assert set(declared) == set(_ffi.EXPORTS), set(declared) ^ set(_ffi.EXPORTS)
  for gone in ("tfrs_inbatch_softmax_tc_ex_workspace_bytes", "tfrs_inbatch_softmax_tc_fwd_ex",
               "tfrs_inbatch_softmax_tc_bwd_ex_workspace_bytes", "tfrs_inbatch_softmax_tc_bwd_ex", "tfrs_topk_merge"):
    assert not hasattr(lib, gone), f"{gone} is still exported"
  # no-compute calls are safe without a GPU
  l = _ffi.lib()
  assert l.tfrs_version() == 102
  assert l.tfrs_topk_scan_workspace_bytes(4096, 1000000, 64, 100) > 0
  assert l.tfrs_launch_count() == 0


def test_sass_is_sm90a_only():
  from recommenders_b200 import build
  out = subprocess.run(["cuobjdump", "-lelf", build.build()], capture_output=True, text=True).stdout
  archs = set(re.findall(r"sm_(\d+a?)", out))
  assert archs == {"90a"}, archs


def test_no_cpu_fallback():
  from recommenders_b200 import ops
  with pytest.raises(RuntimeError, match="CUDA"):
    ops.topk_scan(torch.zeros(2, 4), torch.zeros(8, 4), 3)
  with pytest.raises(RuntimeError, match="CUDA"):
    ops.inbatch_softmax_loss(torch.zeros(2, 4), torch.zeros(2, 4))
  with pytest.raises(RuntimeError, match="CUDA"):
    ops.cross(torch.zeros(2, 4), torch.zeros(2, 4), torch.zeros(4, 4), None)


def test_product_never_imports_oracle():
  """The oracle is test infrastructure: nothing under recommenders_b200/ may import, include, link or load it."""
  pkg = os.path.join(ROOT, "recommenders_b200")
  bad = re.compile(r"(^\s*(from|import)\s+oracle\b)|(#include\s*[\"<][^\">]*oracle)|(libtfrs_oracle)|(oracle\.py)", re.M)
  for dp, _, files in os.walk(pkg):
    for f in files:
      if f.endswith((".py", ".cu", ".cuh")):
        assert not bad.search(open(os.path.join(dp, f)).read()), f


def test_dataset_shim():
  from recommenders_b200.data import Dataset
  x = torch.arange(10).reshape(10, 1).float()
  assert [b.shape[0] for b in Dataset.from_tensor_slices(x).batch(4)] == [4, 4, 2]
  assert [b.shape[0] for b in Dataset.from_tensor_slices(x).batch(4, drop_remainder=True)] == [4, 4]
  ids = np.arange(10).astype(str)
  ds = Dataset.from_tensor_slices((ids, x)).batch(3)
  first = next(iter(ds))
  assert isinstance(first, tuple) and first[0].shape[0] == 3 and first[1].shape == (3, 1)
  assert len(list(ds)) == 4 and len(list(ds)) == 4  # re-iterable
  z = Dataset.zip((Dataset.from_tensor_slices(ids).batch(5), Dataset.from_tensor_slices(x).batch(5)))
  assert [e[0].shape[0] for e in z] == [5, 5]
  m = Dataset.from_tensor_slices(x).batch(5).map(lambda t: t * 2)
  assert float(next(iter(m)).sum()) == 2 * float(x[:5].sum())
  with pytest.raises(ValueError):
    Dataset.from_tensor_slices((ids[:9], x))


def test_metric_accumulators_and_in_top_k():
  from recommenders_b200 import metrics
  m = metrics.Mean("m")
  m.update_state(torch.tensor([[1.0], [0.0]]), torch.tensor([[0.7], [0.3]]))
  assert abs(m.result() - 0.7) < 1e-6
  m.update_state(torch.tensor([1.0, 1.0]))
  assert abs(m.result() - (0.7 + 2.0) / (1.0 + 2.0)) < 1e-6
  m.reset_states()
  assert m.result() == 0.0
  pred = torch.tensor([[0.1, 0.5, 0.5, 0.2], [float("nan"), 1.0, 2.0, 3.0]])
  # tie rule: target counts iff fewer than k predictions are STRICTLY larger; non-finite target -> False
  assert metrics.in_top_k(torch.tensor([1, 0]), pred, 1).tolist() == [True, False]
  assert metrics.in_top_k(torch.tensor([3, 1]), pred, 2).tolist() == [False, False]
  assert metrics.in_top_k(torch.tensor([3, 1]), pred, 3).tolist() == [True, True]
  acc = metrics.TopKCategoricalAccuracy(k=1, name="a")
  acc.update_state(torch.eye(2), torch.tensor([[6.0, 3.0], [9.0, 5.0]]), sample_weight=torch.tensor([0.7, 0.3]))
  assert abs(acc.result() - 0.7) < 1e-6


def test_shard_bounds_cover_the_corpus():
  from recommenders_b200.layers.factorized_top_k import shard_bounds
  for n in (0, 1, 7, 8, 1000003):
    for w in (1, 2, 4, 8):
      b = [shard_bounds(n, r, w) for r in range(w)]
      assert b[0][0] == 0 and b[-1][1] == n
      assert all(b[i][1] == b[i + 1][0] for i in range(w - 1))


_WORKER = r"""
import ctypes, os, sys
import numpy as np, torch, torch.distributed as dist
sys.path.insert(0, os.environ["TFRS_ROOT"])
from oracle import oracle as orc
from recommenders_b200 import _ffi
from recommenders_b200.layers.factorized_top_k import shard_bounds
dist.init_process_group("gloo", init_method="tcp://127.0.0.1:" + os.environ["TFRS_PORT"],
                        rank=int(os.environ["RANK"]), world_size=int(os.environ["WORLD_SIZE"]))
rank, world = dist.get_rank(), dist.get_world_size()
lib = _ffi.lib()
# (1) control plane of ShardComm: rank 0's 128-byte NCCL id reaches every rank unchanged (tfrs_comm_create itself needs GPUs)
uid = (ctypes.c_char * 128)()
if rank == 0:
  assert lib.tfrs_comm_unique_id(uid) == 0, _ffi.last_error()
box = [bytes(uid)]
dist.broadcast_object_list(box, src=0)
digest = torch.tensor([sum(box[0]) + 1000003 * box[0][5]], dtype=torch.int64)
ref = digest.clone(); dist.broadcast(ref, src=0)
assert len(box[0]) == 128 and int(ref) == int(digest), "unique id differs between ranks"
# (2) the data path of tfrs_topk_sharded_f32, byte for byte: every rank writes its local top-k into the packed send
# block [scores f32 [Q,k] | pad | indices i64 [Q,k]] at the offsets the C ABI reports (short shards padded with
# (-inf, INT64_MAX)), ONE all-gather of the blocks, merge reading the receive buffer in place.
rng = np.random.RandomState(0)
N, Q, d, k = 1003, 9, 16, 502      # shard 0 has 502 rows (== k), shard 1 has 501 (< k): the padded case
c = rng.normal(size=(N, d)).astype(np.float32); q = rng.normal(size=(Q, d)).astype(np.float32)
c[700] = c[3]                      # a cross-shard exact tie: the lower global index must win
lo, hi = shard_bounds(N, rank, world)
lay = (ctypes.c_int64 * 4)()
assert lib.tfrs_topk_sharded_layout(world, Q, hi - lo, d, k, lay) == 0
idx_off, block = int(lay[0]), int(lay[1])
blocks = torch.tensor([block], dtype=torch.int64); mx = blocks.clone(); dist.all_reduce(mx, op=dist.ReduceOp.MAX)
assert int(mx) == block, "block size must not depend on the shard"
k_local = min(k, hi - lo)
s, i = orc.topk_scan(q, c[lo:hi], k_local, index_offset=lo)   # the local scan (CUDA kernel on a GPU box)
send = np.zeros(block, dtype=np.uint8)
ss = send[:Q * k * 4].view(np.float32).reshape(Q, k); si = send[idx_off:idx_off + Q * k * 8].view(np.int64).reshape(Q, k)
ss[:] = -np.inf; si[:] = np.iinfo(np.int64).max
ss[:, :k_local] = s; si[:, :k_local] = i
recv = torch.empty(world * block, dtype=torch.uint8)
dist.all_gather_into_tensor(recv, torch.from_numpy(send))
r = recv.numpy()
all_s = np.stack([r[g * block: g * block + Q * k * 4].view(np.float32).reshape(Q, k) for g in range(world)])
all_i = np.stack([r[g * block + idx_off: g * block + idx_off + Q * k * 8].view(np.int64).reshape(Q, k) for g in range(world)])
ms, mi = orc.topk_merge(all_s, all_i, k)               # the merge kernel's oracle
es, ei = orc.topk_scan(q, c, k)
assert np.array_equal(mi, ei) and np.array_equal(ms, es), "sharded result differs from the unsharded scan"
dist.barrier()
print("RANK_OK", rank)
"""


@pytest.mark.parametrize("world", [2])
def test_sharded_protocol_gloo(tmp_path, world):
  script = tmp_path / "worker.py"
  script.write_text(_WORKER)
  port = str(29500 + (os.getpid() % 2000))
  procs = []
  for r in range(world):
    env = {**os.environ, "RANK": str(r), "WORLD_SIZE": str(world), "TFRS_PORT": port, "TFRS_ROOT": ROOT,
           "MASTER_ADDR": "127.0.0.1"}
    procs.append(subprocess.Popen([sys.executable, str(script)], env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True))
  outs = [p.communicate(timeout=240)[0] for p in procs]
  for r, (p, o) in enumerate(zip(procs, outs)):
    assert p.returncode == 0 and f"RANK_OK {r}" in o, o


def test_host_side_planning_functions_with_option_flags():
  """The *_workspace_bytes / out_dim entry points are pure host code: they run without a GPU and define which shapes
  take the tensor-core paths (0 = outside the range, the callers then use the exact kernels)."""
  from recommenders_b200 import _ffi
  lib = _ffi.lib()
  # DotInteraction output width (dot_interaction.py:88-100)
  for F in (1, 2, 3, 27):
    assert lib.tfrs_dot_interaction_out_dim(F, 0, 0) == F * (F - 1) // 2
    assert lib.tfrs_dot_interaction_out_dim(F, 1, 0) == F * (F + 1) // 2
    assert lib.tfrs_dot_interaction_out_dim(F, 0, 1) == F * F and lib.tfrs_dot_interaction_out_dim(F, 1, 1) == F * F
  # in-batch softmax on tensor cores: forward d <= 128, backward d <= 64, C >= B
  assert lib.tfrs_inbatch_softmax_tc_workspace_bytes(16384, 16384, 64, 0, 0) > 0
  assert lib.tfrs_inbatch_softmax_tc_workspace_bytes(16384, 16384, 128, 0, 0) > 0
  assert lib.tfrs_inbatch_softmax_tc_workspace_bytes(16384, 16384, 129, 0, 0) == 0
  assert lib.tfrs_inbatch_softmax_tc_workspace_bytes(1024, 512, 64, 0, 0) == 0
  assert lib.tfrs_inbatch_softmax_tc_bwd_workspace_bytes(16384, 16384, 64, 0, 0) > 0
  assert lib.tfrs_inbatch_softmax_tc_bwd_workspace_bytes(16384, 16384, 65, 0, 0) == 0
  # top-K screening path: k <= 256, d <= 128, corpus large enough
  assert lib.tfrs_topk_tc_workspace_bytes(4096, 1_000_000, 64, 100) > 0
  assert lib.tfrs_topk_tc_workspace_bytes(4096, 1_000_000, 64, 257) == 0
  assert lib.tfrs_topk_tc_workspace_bytes(4096, 1_000_000, 129, 100) == 0
  assert lib.tfrs_topk_tc_workspace_bytes(4096, 1000, 64, 100) == 0
  # workspaces grow with the problem
  assert lib.tfrs_cross_tc_bwd_workspace_bytes(65536, 845) > lib.tfrs_cross_tc_bwd_workspace_bytes(4096, 845) > 0
  assert lib.tfrs_index_bytes(1_000_000, 64) >= 1_000_000 * 64 * 2


def _tree_merge_emulation(scores, idx, k_out):
  """Line-by-line Python restatement of merge_sorted_kernel (csrc/topk.cu): prune every list at
  tau = min_l list_l[rr-1], then merge pairwise in a tree, rank = own position + binary search in the partner list,
  ties between equal (score, index) pairs go to the lower list.  Used to check the ALGORITHM on the CPU; the CUDA
  kernel itself is checked against the sort-based merge and numpy in tests/test_gpu_tc.py."""
  n_lists, k_in = scores.shape
  ko = min(k_out, n_lists * k_in)
  rr = min(k_in, -(-ko // n_lists))
  tau = min(scores[l][rr - 1] for l in range(n_lists))
  lists = []
  for l in range(n_lists):
    n = rr
    while n < k_in and scores[l][n] >= tau:
      n += 1
    lists.append([(float(scores[l][r]), int(idx[l][r])) for r in range(n)])
  if n_lists == 1:
    return lists[0][:ko]

  def precedes(x, e, x_list_is_lower):
    return x[0] > e[0] or (x[0] == e[0] and (x[1] <= e[1] if x_list_is_lower else x[1] < e[1]))

  c_prev = k_in
  while True:
    last = len(lists) <= 2
    c_new = min(ko, 2 * c_prev)
    nxt = [[None] * min(c_new, len(lists[2 * i]) + (len(lists[2 * i + 1]) if 2 * i + 1 < len(lists) else 0))
           for i in range((len(lists) + 1) // 2)]
    for l, lst in enumerate(lists):
      m = l ^ 1
      for r, e in enumerate(lst):
        rank = r
        if m < len(lists):
          lo, hi = 0, len(lists[m])
          while lo < hi:
            mid = (lo + hi) >> 1
            if precedes(lists[m][mid], e, m < l):
              lo = mid + 1
            else:
              hi = mid
          rank += lo
        if rank < c_new:
          assert nxt[l >> 1][rank] is None, "two elements claimed the same merged position"
          nxt[l >> 1][rank] = e
    assert all(x is not None for lst in nxt for x in lst), "a merged position was left empty"
    lists = nxt
    if last:
      return lists[0][:ko]
    c_prev = c_new


def test_sorted_tree_merge_algorithm_matches_a_full_sort():
  """Property test of the pruned tree merge on the CPU: random list counts / lengths / k, heavy score ties, ties
  across lists, (-inf, INT64_MAX) padding of short shards."""
  rng = np.random.default_rng(123)
  for trial in range(300):
    n_lists = int(rng.integers(1, 10)); k_in = int(rng.integers(1, 40)); k_out = int(rng.integers(1, 2 * k_in + 3))
    s = np.round(rng.normal(size=(n_lists, k_in)) * 2) / 2
    i = np.stack([rng.choice(1000, size=k_in, replace=False) for _ in range(n_lists)]).astype(np.int64)
    if trial % 3 == 0:  # distinct index ranges per list, as in the sharded scan
      i += 1000 * np.arange(n_lists)[:, None]
    n_pad = int(rng.integers(0, k_in)) if trial % 4 == 0 else 0
    if n_pad:
      s[-1, k_in - n_pad:] = -np.inf; i[-1, k_in - n_pad:] = np.iinfo(np.int64).max
    for l in range(n_lists):
      order = np.lexsort((i[l], -s[l]))
      s[l], i[l] = s[l][order], i[l][order]
    got = _tree_merge_emulation(s.astype(np.float32), i, k_out)
    flat_s, flat_i = s.reshape(-1).astype(np.float32), i.reshape(-1)
    # expected order: (score desc, index asc), equal pairs in list order -- a stable sort of the concatenation
    order = sorted(range(flat_s.size), key=lambda t: (-flat_s[t], flat_i[t], t))[:min(k_out, flat_s.size)]
    exp = [(float(flat_s[t]), int(flat_i[t])) for t in order]
    assert got == exp, (trial, n_lists, k_in, k_out)


def test_dot_interaction_pair_index_inversion():
  """The forward kernel of csrc/dot_interaction.cu inverts the packed lower-triangle position p -> (i, j) with a
  float sqrt guess and integer correction loops; check that arithmetic (in float32, as on the device) for every
  feature count the kernel accepts."""
  for self_int in (False, True):
    for F in range(1, 65):
      expect = [(a, b) for a in range(F) for b in range(a + 1 if self_int else a)]
      for p, (ei, ej) in enumerate(expect):
        i = int((np.sqrt(np.float32(8.0) * np.float32(p) + np.float32(1.0)) - np.float32(1.0)) * np.float32(0.5))
        if self_int:
          while (i + 1) * (i + 2) // 2 <= p: i += 1
          while i * (i + 1) // 2 > p: i -= 1
          j = p - i * (i + 1) // 2
        else:
          i += 1
          while (i + 1) * i // 2 <= p: i += 1
          while i * (i - 1) // 2 > p: i -= 1
          j = p - i * (i - 1) // 2
        assert (i, j) == (ei, ej), (self_int, F, p)


def _simulate_softmax_bwd_protocol(n_iter, seed, bufs=3, drain=8, stages=4):
  """Randomised interleaving of the barrier protocol of softmax_tc_bwd_kernel (csrc/softmax_tc_bwd.cu): the producer,
  the single MMA-issuing thread (S(it) then dX(it-2), dX chunks drained every `drain` tiles) with its asynchronous but
  in-order tensor pipe, and 16 epilogue warps in two groups.  Barriers are modelled as phase counters; a waiter
  expecting phase k of a barrier may only ever see k or k+1 completed phases (the parity test of mbarrier.try_wait
  cannot tell k+2 from k).  Returns when every agent has finished; raises on deadlock or a phase overrun."""
  import random
  rnd = random.Random(seed)
  done = {}        # barrier name -> completed phases
  arrivals = {}    # barrier name -> arrivals in the current phase
  need = {}        # barrier name -> arrivals per phase

  def bar(name, count):
    done[name] = 0; arrivals[name] = 0; need[name] = count
  for s in range(stages):
    bar(("y_full", s), 1); bar(("y_empty", s), 1)
  for b in range(bufs):
    bar(("s_full", b), 1); bar(("g_ready", b), 8)
  bar("dx_full", 1); bar("dx_drained", 16)

  def arrive(name):
    arrivals[name] += 1
    if arrivals[name] == need[name]:
      arrivals[name] = 0; done[name] += 1

  def ready(name, k):  # may an agent waiting for the k-th completion of `name` proceed?
    assert done[name] <= k + 1, ("phase overrun", name, k, done[name])
    return done[name] >= k + 1

  pipe = []  # in-order queue of commits still to be delivered by the tensor pipe: barrier names

  def producer():
    for it in range(n_iter):
      s = it % stages
      if it >= stages:
        yield (("y_empty", s), it // stages - 1)
      arrive(("y_full", s))  # the bulk copy lands (modelled as immediate)

  def mma():
    def issue_dx(u):
      chunk, first = u // drain, (u % drain) == 0
      if first and chunk > 0:
        yield ("dx_drained", chunk - 1)
      yield (("g_ready", u % bufs), u // bufs)
      pipe.append(("y_empty", u % stages))
      if (u % drain) == drain - 1 or u == n_iter - 1:
        pipe.append("dx_full")
    for it in range(n_iter):
      yield (("y_full", it % stages), it // stages)
      pipe.append(("s_full", it % bufs))
      if it >= 2:
        yield from issue_dx(it - 2)
    if n_iter >= 2:
      yield from issue_dx(n_iter - 2)
    yield from issue_dx(n_iter - 1)

  def epilogue(grp):
    n_chunks = (n_iter + drain - 1) // drain
    state = {"next": 0}

    def drain_until(t_next):
      while state["next"] < n_chunks and min(state["next"] * drain + drain - 1, n_iter - 1) + 3 <= t_next:
        yield ("dx_full", state["next"])
        arrive("dx_drained")
        state["next"] += 1
    for it in range(grp, n_iter, 2):
      yield from drain_until(it)
      yield (("s_full", it % bufs), it // bufs)
      arrive(("g_ready", it % bufs))
    yield from drain_until(n_iter + 3 + drain)

  agents = [producer(), mma()] + [epilogue(w >> 3) for w in range(16)]
  waiting = [None] * len(agents)
  alive = [True] * len(agents)
  for a in range(len(agents)):  # prime
    try:
      waiting[a] = next(agents[a])
    except StopIteration:
      alive[a] = False
  steps = 0
  while any(alive) or pipe:
    steps += 1
    assert steps < 200000, "no progress bound exceeded"
    choices = [a for a in range(len(agents)) if alive[a] and ready(*waiting[a])]
    if pipe:
      choices.append(-1)
    assert choices, ("deadlock", n_iter, seed, [w for w, al in zip(waiting, alive) if al])
    a = rnd.choice(choices)
    if a == -1:
      arrive(pipe.pop(0))  # the tensor pipe retires its oldest batch and its commit arrives
      continue
    try:
      waiting[a] = next(agents[a])
    except StopIteration:
      alive[a] = False
  return steps


def test_softmax_backward_barrier_protocol_has_no_deadlock_or_phase_overrun():
  for n_iter in list(range(1, 40)) + [63, 64, 65, 128]:
    for seed in range(6):
      _simulate_softmax_bwd_protocol(n_iter, seed)


# ------------------------------------------------------------------------------------------------
# Retrieval.call routing (host logic only: the kernels are replaced by recorders, tensors stay on the CPU)
# ------------------------------------------------------------------------------------------------
def _routing_case(monkeypatch, supported=True):
  import torch
  from recommenders_b200 import ops, tasks
  calls = []

  def rec(name):
    def f(*a, **k):
      calls.append((name, a, k))
      return torch.zeros((), requires_grad=True)
    return f
  monkeypatch.setattr(ops, "inbatch_softmax_loss", rec("fused"))
  monkeypatch.setattr(ops, "hard_negative_softmax_loss", rec("hardneg"))
  monkeypatch.setattr(ops, "inbatch_softmax_maxsim_loss", rec("maxsim"))
  monkeypatch.setattr(ops, "inbatch_softmax_bias_supported", lambda B, C, d: supported)
  monkeypatch.setattr(ops, "hard_negative_supported", lambda B, C, d, n: supported)
  monkeypatch.setattr(ops, "scores", lambda q, c: (calls.append(("scores", (q, c), {})), q @ c.T)[1])
  return tasks, calls


def test_retrieval_routes_loss_options_to_fused_kernels(monkeypatch):
  import torch
  tasks, calls = _routing_case(monkeypatch)
  q, c = torch.randn(8, 4), torch.randn(12, 4)
  ids = torch.arange(12); mask = torch.ones(8, 12, dtype=torch.bool); prob = torch.full((12,), 0.1)
  tasks.Retrieval()(q, c, compute_metrics=False)
  assert [n for n, *_ in calls] == ["fused"] and calls[-1][1][4:] == ()          # plain: no options passed
  calls.clear()
  tasks.Retrieval(temperature=0.5, remove_accidental_hits=True)(q, c, candidate_ids=ids, score_mask=mask,
                                                                candidate_sampling_probability=prob, compute_metrics=False)
  (name, a, _), = calls
  assert name == "fused" and a[3] == 0.5 and a[4] is not None and a[5] is ids and a[6] is not None
  assert torch.allclose(a[4], -torch.log(prob))                                   # the correction travels as a bias vector
  calls.clear()
  tasks.Retrieval(remove_accidental_hits=False)(q, c, candidate_ids=ids, score_mask=mask, compute_metrics=False)
  assert calls[0][1][5] is None                                                   # ids given but the option is off: not used
  calls.clear()
  tasks.Retrieval(num_hard_negatives=3, temperature=2.0)(q, c, compute_metrics=False)
  assert [n for n, *_ in calls] == ["hardneg"] and calls[0][1][2] == 3
  calls.clear()
  tasks.Retrieval()(torch.randn(8, 2, 4), c, compute_metrics=False)
  assert [n for n, *_ in calls] == ["maxsim"]


def test_retrieval_falls_back_to_the_reference_sequence_when_needed(monkeypatch):
  import torch
  tasks, calls = _routing_case(monkeypatch, supported=False)
  q, c = torch.randn(8, 4), torch.randn(12, 4)
  ids = torch.arange(12)
  # shapes outside the tensor-core range: the options run on the exact score matrix, in the reference's order
  loss = tasks.Retrieval(remove_accidental_hits=True, num_hard_negatives=2)(q, c, candidate_ids=ids, compute_metrics=False)
  assert [n for n, *_ in calls] == ["scores"] and loss.dim() == 0
  calls.clear()
  # hard negatives combined with a mask, a custom loss object, or batch metrics always need the logits
  tasks2, calls2 = _routing_case(monkeypatch, supported=True)
  tasks2.Retrieval(num_hard_negatives=2)(q, c, score_mask=torch.ones(8, 12, dtype=torch.bool), compute_metrics=False)
  assert [n for n, *_ in calls2] == ["scores"]
  calls2.clear()
  tasks2.Retrieval(loss=lambda y, s, w=None: s.sum())(q, c, compute_metrics=False)
  assert [n for n, *_ in calls2] == ["scores"]
  calls2.clear()
  tasks2.Retrieval(num_hard_negatives=2, temperature=-1.0)(q, c, compute_metrics=False)   # order-reversing temperature
  assert [n for n, *_ in calls2] == ["scores"]
  with pytest.raises(ValueError):
    tasks2.Retrieval(remove_accidental_hits=True)(q, c, compute_metrics=False)


def test_candidate_ids_of_any_type_become_int64_codes():
  """Accidental-hit removal only needs EQUALITY of ids: strings / object arrays / float ids are factorised on the host."""
  import numpy as np
  import torch
  from recommenders_b200 import ops
  dev = torch.device("cpu")
  s = np.asarray(["b", "a", "b", "c", "a"])
  codes = ops._ids_i64(s, 5, dev)
  assert codes.dtype == torch.int64 and codes[0] == codes[2] and codes[1] == codes[4] and len(set(codes.tolist())) == 3
  t = torch.tensor([7, 7, 2 ** 40 + 1, 2 ** 40 + 1, -3])
  assert torch.equal(ops._ids_i64(t, 5, dev), t)                       # integer tensors are used as they are
  f = torch.tensor([0.5, 1.5, 0.5, 2.0, 1.5])
  cf = ops._ids_i64(f, 5, dev)
  assert cf[0] == cf[2] and cf[1] == cf[4] and cf[3] != cf[0]
  with pytest.raises(ValueError):
    ops._ids_i64(s, 6, dev)


def test_bucketed_rank_sort_groups_ids_in_order_of_occurrence():
  """CPU model of csrc/adagrad.cu's bucketed rank sort: whatever order the scatter's atomics produce inside a bucket, the
  ranks (number of bucket members below a key) place every id's members contiguously and in order of occurrence -- all the
  segmented Adagrad update needs -- and the result does not depend on the scatter order."""
  import numpy as np
  rng = np.random.RandomState(3)

  def bucket(key):
    idv = ((key >> np.uint64(24)) ^ (key >> np.uint64(56))).astype(np.uint32)
    return ((idv.astype(np.uint64) * np.uint64(0x9E3779B1)) & np.uint64(0xFFFFFFFF)).astype(np.uint32) >> np.uint32(24)

  def sort_once(ids, seed):
    n = len(ids)
    keys = (ids.astype(np.uint64) << np.uint64(24)) | np.arange(n, dtype=np.uint64)
    b = bucket(keys)
    order = np.random.RandomState(seed).permutation(n)           # the nondeterministic part: arrival order of the atomics
    bkeys, bstart = [], [0]
    for v in range(256):
      m = order[b[order] == v]
      bkeys.extend(keys[m]); bstart.append(len(bkeys))
    bkeys = np.asarray(bkeys, np.uint64)
    out = np.zeros(n, np.uint64)
    for v in range(256):
      seg = bkeys[bstart[v]:bstart[v + 1]]
      for key in seg:
        out[bstart[v] + int((seg < key).sum())] = key             # rank inside the bucket (keys are unique)
    return out

  for ids in (rng.randint(0, 50, size=700), rng.randint(0, 10 ** 9, size=900), np.zeros(300, np.int64),
              (rng.zipf(1.3, size=800) % 1000)):
    ids = np.asarray(ids, np.int64)
    a, b2 = sort_once(ids, 1), sort_once(ids, 2)
    assert np.array_equal(a, b2)                                   # deterministic despite the scatter order
    assert np.array_equal(np.sort(a), np.sort((ids.astype(np.uint64) << np.uint64(24)) | np.arange(len(ids), dtype=np.uint64)))
    out_ids = (a >> np.uint64(24)).astype(np.int64); pos = (a & np.uint64(0xFFFFFF)).astype(np.int64)
    seen = set()
    for i in range(len(a)):
      if i and out_ids[i] == out_ids[i - 1]:
        assert pos[i] > pos[i - 1]                                 # members in order of occurrence
      else:
        assert out_ids[i] not in seen                              # every id forms ONE contiguous run
        seen.add(out_ids[i])


def test_workspace_cache_is_bounded(monkeypatch):
  """_ffi.workspace keeps at most _WS_CACHE_MAX buffers (least recently used dropped) and grows a slot on demand."""
  import torch
  from recommenders_b200 import _ffi

  class _S:
    cuda_stream = 0
  made = []
  monkeypatch.setattr(torch.cuda, "current_stream", lambda *a, **k: _S())
  monkeypatch.setattr(torch.cuda, "current_device", lambda: 0)
  real_empty = torch.empty
  monkeypatch.setattr(torch, "empty", lambda n, dtype=None, device=None: (made.append(n), real_empty(n, dtype=dtype))[1])
  _ffi.release_workspaces()
  dev = torch.device("cpu")
  a = _ffi.workspace(1000, dev, "a")
  assert _ffi.workspace(500, dev, "a") is a and len(made) == 1          # reused while large enough
  assert _ffi.workspace(5000, dev, "a").numel() >= 5000 and len(made) == 2
  for i in range(_ffi._WS_CACHE_MAX + 10):
    _ffi.workspace(256, dev, f"slot{i}")
    _ffi.workspace(256, dev, "a")                                         # keeps "a" recent
  assert len(_ffi._ws_cache) == _ffi._WS_CACHE_MAX and any(k[2] == "a" for k in _ffi._ws_cache)
  assert not any(k[2] == "slot0" for k in _ffi._ws_cache)
  _ffi.release_workspaces()
  assert not _ffi._ws_cache
