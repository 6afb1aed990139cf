"""The survivor records of the tensor-core top-K filter pass (csrc/topk_tc.cu, tc_scan_kernel<FILTER>), read out of the
call's workspace and checked exactly.

Queries and corpus hold small integers, so every screening product and sum is exact in fp16 x fp16 -> fp32 whatever the
accumulation order, and the power-of-two rescale is exact: the screening score of (query, column) is known bit for bit.
For every (query, corpus part, column half) segment the live records must be exactly the octets of that part's tiles
with a screening score >= the query's filter threshold, in ascending column order, with the 8 rescaled scores of the
octet (the zero-padded rows of the last tile score 0) and the right count.
"""
import ctypes
import math

import pytest
import torch

from test_gpu_topk_tc_edges import _tc_rows

pytestmark = pytest.mark.gpu

TILE = 128


@pytest.fixture(scope="module")
def ops():
  from recommenders_b200 import ops as o
  return o


def _ints(shape, seed):
  g = torch.Generator(device="cuda"); g.manual_seed(seed)
  return torch.randint(-32, 33, shape, generator=g, device="cuda").to(torch.float32)


@pytest.mark.parametrize("Q,N,k", [(500, 201 * TILE - 91, 32), (256, 64 * TILE + 5, 16)])
def test_filter_records_exact(ops, Q, N, k):
  d = 64
  q, c = _ints((Q, d), 11), _ints((N, d), 12)
  # Query 0's best possible corpus row, planted at octets 0, 1 and 3 of half 0 and octet 7 of half 1 of two tiles.  These
  # 8 rows are query 0's best scores (k >= 8), so one (row, tile, half) has several surviving octets, not all adjacent:
  # the records of one quad take more than one pass of the set-bit walk.
  n_tiles = -(-N // TILE)
  best = 32.0 * torch.sign(q[0])
  for t in (0, n_tiles // 2):
    for col in (0, 8, 24, 64 + 56):
      c[t * TILE + col] = best
  assert ops.tc_supported(Q, N, d, k)
  idx = ops.index_build(c)
  s, i = ops.topk_tc(q, c, idx, k)
  es, ei = ops.topk_scan(q, c, k)
  assert torch.equal(i, ei) and torch.equal(s.view(torch.int32), es.view(torch.int32))

  rows = _tc_rows(ops, Q, N, d, k)   # per-row state (threshold, exponent, fallback), checked against the restated plan
  assert not rows["fallback"].any(), "a row took the exact fallback"
  assert not rows["seg_ovf"].any(), "a segment overflowed: choose data with fewer survivors per segment"
  # the record arrays, at the same layout offsets _tc_rows reads
  out = (ctypes.c_int64 * 10)()
  ops.check(ops.lib().tfrs_topk_tc_layout(Q, N, d, k, out), "topk_tc_layout")
  o_count, _, _, o_cand, segs, cap, Qp = [int(x) for x in out[:7]]
  dev = q.device
  ws = ops.workspace(0, dev, "tc")
  base = (-ws.data_ptr()) % 16

  def arr(off, n, dtype):
    return ws[base + off: base + off + 4 * n].view(dtype)

  count = arr(o_count, Qp * segs, torch.int32).view(Qp, segs)[:Q].to(torch.int64)
  cand_s = arr(o_cand, Qp * segs * cap * 8, torch.float32).view(Qp, segs, cap, 8)[:Q]
  cand_i = arr(o_cand + Qp * segs * cap * 32, Qp * segs * cap, torch.int32).view(Qp, segs, cap)[:Q].to(torch.int64)
  assert torch.equal(count.sum(1).cpu(), torch.from_numpy(rows["records"]).to(torch.int64))
  thr = torch.from_numpy(rows["thr"]).to(dev)
  qexp = torch.from_numpy(rows["qexp"]).to(dev).to(torch.float64)
  cexp = 15.0 - math.frexp(float(c.abs().max()))[1]   # the corpus exponent: largest |c| * 2^e lands in [2^14, 2^15)

  parts = segs // 2
  assert parts >= 2, "the shape must split the corpus over several parts"
  cz = torch.zeros((n_tiles * TILE, d), dtype=torch.float64, device=dev)
  cz[:N] = c.double()
  screen = torch.ldexp(q.double() @ cz.T, (cexp + qexp)[:, None]).to(torch.float32)   # exact: integers times 2^e
  octet = screen.view(Q, n_tiles, 2, 8, 8)                                            # [q, tile, half, j, column]
  hit = (octet >= thr[:, None, None, None, None]).any(-1)                             # [q, tile, half, j]
  for t in (0, n_tiles // 2):
    assert hit[0, t, 0, [0, 1, 3]].all() and hit[0, t, 1, 7], "the planted octets must survive"

  for part in range(parts):
    t0, t1 = part * n_tiles // parts, (part + 1) * n_tiles // parts
    for h in range(2):
      seg = 2 * part + h
      hm = hit[:, t0:t1, h, :].reshape(Q, -1)              # octets in ascending column order
      assert torch.equal(count[:, seg], hm.sum(1)), (part, h)
      cols = (torch.arange(t0, t1, device=dev)[:, None] * TILE + 64 * h + 8 * torch.arange(8, device=dev)).reshape(-1)
      qi, ki = hm.nonzero(as_tuple=True)
      pos = (hm.cumsum(1) - 1)[qi, ki]
      assert torch.equal(cand_i[qi, seg, pos], cols[ki]), (part, h)
      want = octet[:, t0:t1, h].reshape(Q, -1, 8)[qi, ki]
      assert torch.equal(cand_s[qi, seg, pos].view(torch.int32), want.view(torch.int32)), (part, h)
