"""The REAL sharded path: two processes, two GPUs, NCCL issued by libtfrs_b200.so (tfrs_comm_* / tfrs_topk_sharded_f32),
compared with the oracle and with the unsharded exact scan.  Skipped on boxes with fewer than 2 GPUs
(`python -m pytest tests/test_gpu_multi.py -m gpu` on a machine with two GPUs runs it)."""
import os
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

_WORKER = r"""
import ctypes, os, sys
import numpy as np, torch, torch.distributed as dist
sys.path.insert(0, os.environ["TFRS_ROOT"])
import recommenders_b200 as tfrs
from recommenders_b200 import ops, _ffi
from recommenders_b200.layers.factorized_top_k import shard_bounds, ShardComm
from oracle import oracle as orc
rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
torch.cuda.set_device(int(os.environ["LOCAL_RANK"]))
dev = torch.device("cuda", int(os.environ["LOCAL_RANK"]))
dist.init_process_group("gloo")            # control plane only: the data path's NCCL lives behind the C ABI
comm = ShardComm()
def gen(shape, seed):
  g = torch.Generator(device=dev); g.manual_seed(seed)
  return torch.randn(shape, generator=g, device=dev)
# (a) tensor-core shards, (b) exact-path shards with the last shard SHORTER than k (padded blocks), (c) d = 128
for name, N, d, Q, k in (("tc", 200_003, 64, 1000, 100), ("short", 1001, 32, 50, 600), ("d128", 150_000, 128, 300, 50)):
  c = gen((N, d), 1); q = gen((Q, d), 2)
  c[N - 5] = c[3]                           # a cross-shard exact tie: the lower global index must win
  lo, hi = shard_bounds(N, rank, world)
  layer = tfrs.layers.factorized_top_k.BruteForce(k=k).index_shard(c[lo:hi], lo, comm=comm)
  s, i = layer(q)
  es, ei = ops.topk_scan(q, c, k)           # the unsharded exact scan on this rank's own copy
  assert torch.equal(i.to(torch.int64), ei) and torch.equal(s, es), name + ": sharded != unsharded"
  os_, oi = orc.topk_scan(q[:4].cpu().numpy(), c.cpu().numpy(), k)
  assert np.array_equal(i[:4].cpu().numpy(), oi) and np.array_equal(s[:4].cpu().numpy(), os_), name + ": != oracle"
# the raw collective of the ABI: every rank's [Q,k] lists in rank order
Q, k = 64, 10
s = torch.full((Q, k), float(rank), device=dev); i = torch.full((Q, k), rank * 1000, dtype=torch.int64, device=dev)
all_s = torch.empty((world, Q, k), device=dev); all_i = torch.empty((world, Q, k), dtype=torch.int64, device=dev)
_ffi.check(_ffi.lib().tfrs_topk_allgather(comm.handle, _ffi.ptr(s), _ffi.ptr(i), Q, k, _ffi.ptr(all_s), _ffi.ptr(all_i), _ffi.stream()), "allgather")
torch.cuda.synchronize()
for r in range(world):
  assert float(all_s[r].min()) == float(all_s[r].max()) == float(r) and int(all_i[r].max()) == r * 1000
comm.close()
dist.barrier()
open(os.path.join(os.environ["TFRS_OK_DIR"], f"ok_{rank}"), "w").write("ok")   # a file per rank: stdout of two ranks interleaves
"""


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_sharded_bruteforce_two_gpus(tmp_path):
  script = tmp_path / "worker.py"
  script.write_text(_WORKER)
  port = str(29600 + (os.getpid() % 1000))
  env = {**os.environ, "TFRS_ROOT": ROOT, "TFRS_OK_DIR": str(tmp_path)}
  cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
         "--master-port", port, str(script)]
  r = subprocess.run(cmd, env=env, capture_output=True, text=True, timeout=600)
  done = all((tmp_path / f"ok_{rank}").exists() for rank in (0, 1))
  assert r.returncode == 0 and done, r.stdout[-3000:] + r.stderr[-3000:]
