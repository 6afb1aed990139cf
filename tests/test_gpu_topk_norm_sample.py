"""The norm sample of the tensor-core top-K scan (csrc/topk_tc.cu): from 2^19 rows the index also holds an image of the
floor(N/8) rows of largest norm (whole tiles, index order, ties to the lower index), and takes it as the sampled pass's
sample when the random-direction model gives it phi >= 0.35 and probe queries made of corpus rows find enough of their
neighbours in it.  Its threshold is the k-th bin bound for both the filter
and the guarantee, so no row retries.  Checked: the choice through the header, the image bytes, the thresholds bit for
bit on exactly screened data, and the results of every mode against the exact scan and the oracle.
"""
import ctypes
import math

import numpy as np
import pytest
import torch
from scipy.special import erfc
from scipy.optimize import brentq

from test_gpu_topk_tc_edges import TILE, _cdiv, _check_topk, _tc_rows
from test_gpu_topk_stat_threshold import _retry_rows
from oracle import oracle as orc

pytestmark = pytest.mark.gpu

HEADER = 1024
SAMPLE_OFF, PHI_OFF = 28, 48   # IndexHeader: SideStats (16 B), d, d_pad, kb, sample; n, n_tiles; phi, probe mean, min


@pytest.fixture(scope="module")
def ops():
  from recommenders_b200 import ops as o
  return o


def _header(image):
  h = image[:HEADER].cpu().numpy()
  return int(h[SAMPLE_OFF:SAMPLE_OFF + 4].view(np.int32)[0]), float(h[PHI_OFF:PHI_OFF + 4].view(np.float32)[0])


def _gauss(N, d, seed):
  g = torch.Generator(device="cuda"); g.manual_seed(seed)
  return torch.randn((N, d), generator=g, device="cuda")


def _rows_of_image(img, tiles, kb):
  """[tiles * 128, kb * 128] bytes of a tile image, the 128-byte swizzle undone (each row's fp16 values in order)."""
  a = img[:tiles * kb * 16384].cpu().numpy().reshape(tiles, kb, 128, 8, 16)
  r = np.arange(128)[:, None]
  a = a[:, :, r, np.arange(8)[None, :] ^ (r & 7)]              # [tiles, kb, 128, 8, 16]
  return a.transpose(0, 2, 1, 3, 4).reshape(tiles * 128, kb * 128)


def _sample_layout(ops, Q, N, d, k):
  out = (ctypes.c_int64 * 8)()
  ops.check(ops.lib().tfrs_topk_tc_sample_layout(Q, N, d, k, out), "topk_tc_sample_layout")
  return dict(zip(("o_binmax", "bins_ld", "n_bins", "group", "bpp", "parts", "tiles", "o_margin"), (int(x) for x in out)))


def _phi(norms, S):
  """The random-direction model restated: t solves sum P(r_i g > t) = N 1e-4; phi = the top-S rows' share of it."""
  r = np.sort(norms.astype(np.float64))[::-1]
  r = r[r > 0]
  target = len(norms) * 1e-4
  f = lambda t: (0.5 * erfc(t / (r * math.sqrt(2)))).sum() - target
  t = brentq(f, 0.0, 40.0 * r[0])
  return (0.5 * erfc(t / (r[:S] * math.sqrt(2)))).sum() / target


@pytest.fixture(scope="module")
def gauss_1m(ops):
  c = _gauss(1_000_000, 64, 1)
  return c, ops.index_build(c)


def test_sample_choice(ops, gauss_1m):
  c, image = gauss_1m
  mode, phi = _header(image)
  probe_mean, probe_min = image[PHI_OFF + 4:PHI_OFF + 12].cpu().numpy().view(np.float32)
  assert mode == 1 and probe_mean >= 0.35 and probe_min >= 0.25, (phi, probe_mean, probe_min)
  S = 1_000_000 // 8 // TILE * TILE
  assert abs(phi - _phi(c.double().norm(dim=1).cpu().numpy(), S)) < 2e-3, phi
  assert ops.lib().tfrs_index_bytes(1_000_000, 64) == HEADER + (_cdiv(1_000_000, TILE) + S // TILE) * 16384
  unit = c / c.norm(dim=1, keepdim=True)
  assert _header(ops.index_build(unit))[0] == 0
  two = unit.clone(); two[::2] *= 2.0                  # two norm levels, half and half: phi ~ 0.25
  assert _header(ops.index_build(two))[0] == 0
  N = (1 << 19) - TILE
  assert ops.lib().tfrs_index_bytes(N, 64) == HEADER + N // TILE * 16384
  assert _header(ops.index_build(_gauss(N, 64, 3)))[0] == 0


def _int_corpus(N, d, seed):
  """Small integers times a per-row scale in {1, 2, 3, 4}: every norm^2 is an exact integer (ties at the cutoff) and
  every screening score is exact."""
  g = torch.Generator(device="cuda"); g.manual_seed(seed)
  c = torch.randint(-8, 9, (N, d), generator=g, device="cuda").float()
  s = torch.randint(1, 5, (N, 1), generator=g, device="cuda").float()
  return c * s


def _expected_sample(c, S):
  n2 = (c.double() ** 2).sum(1).cpu().numpy()
  order = np.lexsort((np.arange(len(n2)), -n2))       # norm desc, index asc
  return np.sort(order[:S])


@pytest.mark.parametrize("N", [1 << 19, 1_000_000])
def test_sample_image_and_thresholds(ops, N):
  Q, d, k = 256, 64, 100
  c = _int_corpus(N, d, 7 + N % 5)
  g = torch.Generator(device="cuda"); g.manual_seed(8)
  q = torch.randint(-32, 33, (Q, d), generator=g, device="cuda").float()
  image = ops.index_build(c)
  assert _header(image)[0] == 1
  lay = _sample_layout(ops, Q, N, d, k)
  S = N // 8 // TILE * TILE
  assert lay["tiles"] * TILE == S and lay["n_bins"] > 0
  rows = _expected_sample(c, S)
  n_tiles = _cdiv(N, TILE)
  main = _rows_of_image(image[HEADER:], n_tiles, 1)
  samp = _rows_of_image(image[HEADER + n_tiles * 16384:], S // TILE, 1)
  np.testing.assert_array_equal(samp, main[rows])

  _check_topk(ops, q, c, k)
  st = _tc_rows(ops, Q, N, d, k)
  safe, retry = _retry_rows(ops, Q, N, d, k)
  assert not st["fallback"].any() and not retry.any()
  np.testing.assert_array_equal(st["thr"].view(np.uint32), safe.view(np.uint32))
  # bin maxima restated from the sample rows: each part's sample tiles in groups, one bin per group and column half
  dots = q.double().cpu().numpy() @ c.double().cpu().numpy()[rows].T
  bins = []
  for p in range(lay["parts"]):
    u0, u1 = p * lay["tiles"] // lay["parts"], (p + 1) * lay["tiles"] // lay["parts"]
    for b0 in range(u0, u1, lay["group"]):
      for h in range(2):
        cols = (np.arange(b0, min(b0 + lay["group"], u1))[:, None] * TILE + 64 * h + np.arange(64)).reshape(-1)
        bins.append(dots[:, cols].max(1))
  bm = -np.sort(-np.stack(bins, 1), axis=1)
  assert bm.shape[1] <= lay["n_bins"]
  ws = ops.workspace(0, torch.device("cuda", torch.cuda.current_device()), "tc")
  base = (-ws.data_ptr()) % 16
  margin = ws[base + lay["o_margin"]: base + lay["o_margin"] + 4 * Q].view(torch.float32).cpu().numpy()
  unit = np.ldexp(1.0, 15 - math.frexp(32.0)[1] + st["qexp"].astype(np.int64))
  L_k = (bm[:, k - 1] * unit).astype(np.float32)
  np.testing.assert_array_equal(safe.view(np.uint32), (L_k - margin).view(np.uint32))


def test_modes_match_exact(ops, gauss_1m):
  c, image = gauss_1m
  Q, k, E = 512, 100, 4
  q = _gauss(Q, 64, 2)
  s, i = ops.topk_tc(q, c, image, k)
  st = ops.tc_last_call_stats(Q, c.shape[0], 64, k)
  assert st["fallback_queries"] == 0, st
  _, retry = _retry_rows(ops, Q, c.shape[0], 64, k)
  assert not retry.any()
  es, ei = ops.topk_scan(q, c, k)
  assert torch.equal(i, ei) and torch.equal(s.view(torch.int32), es.view(torch.int32))
  os_, oi = orc.topk_scan(q[:4].cpu().numpy(), c.cpu().numpy(), k)
  np.testing.assert_array_equal(i[:4].cpu().numpy(), oi)
  ex = torch.stack([i[:, j] for j in (0, 3, 50, 99)], 1)
  xs, xi = ops.topk_tc_exclude(q, c, image, k, ex)
  fs, fi = ops.topk_scan(q, c, k + E)
  cs, ci = orc.exclude(fs.cpu().numpy(), fi.cpu().numpy(), ex.cpu().numpy(), k)
  np.testing.assert_array_equal(xi.cpu().numpy(), ci)
  np.testing.assert_array_equal(xs.cpu().numpy().view(np.uint32), cs.view(np.uint32))
  pos = torch.where(torch.arange(Q, device="cuda") % 2 == 0, es[:, 40], ops.rowwise_dot(q, c[:Q]))
  cnt = ops.topk_tc_count(q, c, image, k, pos)
  np.testing.assert_array_equal(cnt.cpu().numpy(), np.minimum((es > pos[:, None]).sum(1).cpu().numpy(), k))


def test_bruteforce_and_shards(ops):
  import recommenders_b200 as tfrs
  N = 1 << 20
  c = _gauss(N, 64, 21); q = _gauss(300, 64, 22)
  layer = tfrs.layers.factorized_top_k.BruteForce(k=100).index(c)
  assert _header(layer._tc_index)[0] == 1
  s, i = layer(q)
  es, ei = ops.topk_scan(q, c, 100)
  assert torch.equal(i.to(torch.int64), ei) and torch.equal(s, es)
  parts = []
  for lo, hi in (tfrs.layers.factorized_top_k.shard_bounds(N, r, 2) for r in range(2)):
    l = tfrs.layers.factorized_top_k.BruteForce(k=100).index(c[lo:hi])
    assert _header(l._tc_index)[0] == 1
    parts.append(l._local_topk(q, 100, lo))
  ms, mi = ops.topk_merge(torch.stack([p[0] for p in parts]), torch.stack([p[1] for p in parts]), 100)
  assert torch.equal(mi, ei) and torch.equal(ms, es)


def test_high_norm_rows_orthogonal_to_queries(ops):
  """The sample's rows (norm 20) live in dims 0-7, every query in dims 8-63: each sample score is 0, so the bound is
  valid but loose.  The answer stays exact, on the tensor cores or in the fallback, and the call leaves the index as it
  was."""
  N, Q, d, k = 1 << 19, 128, 64, 100
  c = _gauss(N, d, 31) * 0.25                          # small enough that the sample holds every probe's neighbours
  big = torch.arange(0, N, 4, device="cuda")[: N // 8]
  c[big] = 0.0
  c[big, :8] = _gauss(len(big), 8, 32)
  c[big, :8] *= 20.0 / c[big, :8].norm(dim=1, keepdim=True)
  q = _gauss(Q, d, 33); q[:, :8] = 0.0
  image = ops.index_build(c)
  assert _header(image)[0] == 1
  before = image.clone()
  s, i = ops.topk_tc(q, c, image, k)
  es, ei = ops.topk_scan(q, c, k)
  assert torch.equal(i, ei) and torch.equal(s.view(torch.int32), es.view(torch.int32))
  assert torch.equal(image, before), "a query call must not write the index"


def test_clustered_corpus_keeps_the_strided_sample(ops):
  """tools/bench_tree_ah.py's mixture (4096 centers N(0, 1), rows = center + 0.35 N(0, 1)): the norms alone look like an
  iso Gaussian corpus's (phi >= 0.35), but a query near a center has its neighbours in its own cluster, which the norm
  sample holds for few clusters.  The probes see it, and the index keeps the strided sample."""
  N, d = 1_000_000, 64
  g = torch.Generator(device="cuda"); g.manual_seed(5)
  centers = torch.randn((4096, d), generator=g, device="cuda")
  c = centers[torch.randint(0, 4096, (N,), generator=g, device="cuda")] + 0.35 * torch.randn((N, d), generator=g, device="cuda")
  h = ops.index_build(c)[:HEADER].cpu().numpy()
  phi, probe_mean, probe_min = h[PHI_OFF:PHI_OFF + 12].view(np.float32)
  assert phi >= 0.35 and probe_min < 0.25, (phi, probe_mean, probe_min)
  assert int(h[SAMPLE_OFF:SAMPLE_OFF + 4].view(np.int32)[0]) == 0
