"""K19 (GRU) and K20 (LSTM) recurrence kernels on the H100, called through the C ABI with float32 gx, U and saved tensors
the test chooses, each direction per element against its own float64 oracle (tests/gru_oracle.py, tests/lstm_oracle.py):
the forward from gx, the reverse from the oracle's saved tensors rounded to float32.  Bars are 2 u_r times the
first-order bound of tests/rnn_error.py; what the header defines exactly is compared bit for bit:
  - at a masked step out_seq repeats h_{t-1}, h_prev and c_seq carry, and the dgx / dz row is +0;
  - a fully masked row's h_T / c_T are h0 / c0, its dh0 the float32 sum from +0 of g_seq[T-1], g_last, g_seq[T-2], ...,
    g_seq[0], and its dc0 is +0 + g_c;
  - every output is written (no NaN sentinel left) except the gates of masked steps (left alone), and the guard words
    after every buffer are untouched;
  - a row's NaN / Inf reaches no other row, wherever it sits in its CTA.
The cases (tests/rnn_edge_cases.py) reach every (cell, direction, UJ, mask type) instance, the resident / streamed flips,
the slice edges, the batch and length edges and the special mask values."""
import ctypes

import numpy as np
import pytest
import torch

import gru_oracle as go
import lstm_oracle as lo
import rnn_edge_cases as ec
import rnn_error as re_
from recommenders_b200 import _ffi

pytestmark = pytest.mark.gpu

SENTINEL = 0x7FC5A5A5          # a quiet NaN no kernel computes
GUARD = 0x5A5A5A5A
GUARD_WORDS = 64
KIND_CODE = {"bool": _ffi.BOOL, "int32": _ffi.I32, "int64": _ffi.I64}
TORCH_MASK = {"bool": torch.bool, "int32": torch.int32, "int64": torch.int64}
WORST = {}                     # (cell, direction) -> (err / bar, case)


@pytest.fixture(scope="module", autouse=True)
def _report():
  yield
  for k, (r, name) in sorted(WORST.items()):
    print(f"worst err/bar {k[0]} {k[1]}: {r:.4f} ({name})")


class Buf:
  """An output of `shape` float32 elements filled with the NaN sentinel, followed by GUARD_WORDS guard words."""

  def __init__(self, shape):
    self.shape, self.n = tuple(shape), int(np.prod(shape))
    self.raw = torch.full((self.n + GUARD_WORDS,), SENTINEL, dtype=torch.int32, device="cuda")
    self.raw[self.n:] = GUARD

  @property
  def p(self):
    return ctypes.c_void_p(self.raw.data_ptr())

  def bits(self):
    return self.raw[:self.n].cpu().numpy().reshape(self.shape)

  def f32(self):
    return self.bits().view(np.float32)

  def guard_ok(self):
    return bool((self.raw[self.n:] == GUARD).all())


def _dev(a):
  return None if a is None else torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _p(t):
  return None if t is None else ctypes.c_void_p(t.data_ptr())


def _mask_dev(d, kind):
  if kind is None:
    return None, 0
  return torch.from_numpy(np.ascontiguousarray(d["mask"])).cuda().to(TORCH_MASK[kind]), KIND_CODE[kind]


def run_fwd(cell, d, kind, opts):
  """the forward kernel on d's gx, U, (b_r), h0, (c0) and mask: dict of Buf"""
  B, T, nu = d["gx"].shape
  u = nu // ec.NG[cell]
  gx, U, h0, br, c0 = (_dev(d.get(n)) for n in ("gx", "U", "h0", "b_r", "c0"))   # held until the kernel has run
  m, mk = _mask_dev(d, kind)
  o = {"seq": Buf((B, T, u)) if opts["seq"] else None, "h_T": Buf((B, u)), "gates": Buf((B, T, 4 * u)),
       "h_prev": Buf((B, T, u))}
  seq = o["seq"].p if o["seq"] else None
  lib = _ffi.lib()
  if cell == "gru":
    rc = lib.tfrs_gru_fwd_f32(_p(gx), _p(U), _p(br), _p(h0), _p(m), mk, B, T, u, seq, o["h_T"].p, o["gates"].p,
                              o["h_prev"].p, _ffi.stream())
  else:
    o["c_T"], o["c_seq"] = Buf((B, u)), Buf((B, T, u))
    rc = lib.tfrs_lstm_fwd_f32(_p(gx), _p(U), _p(h0), _p(c0), _p(m), mk, B, T, u, seq, o["h_T"].p, o["c_T"].p,
                               o["gates"].p, o["c_seq"].p, o["h_prev"].p, _ffi.stream())
  _ffi.check(rc, f"{cell}_fwd")
  torch.cuda.synchronize()
  return {k: v for k, v in o.items() if v is not None}


def run_bwd(cell, d, saved, kind, opts, dU=False):
  """the reverse kernel on the saved tensors (float32 arrays) and d's upstream gradients: dict of Buf (+ dU, db_r)"""
  B, T, u = saved["h_prev"].shape
  ng = ec.NG[cell]
  U, gates, h_prev, c_seq = _dev(d["U"]), _dev(saved["gates"]), _dev(saved["h_prev"]), _dev(saved.get("c_seq"))
  c0, g_seq, g_last, g_c = (_dev(d.get(n)) for n in ("c0", "g_seq", "g_last" if cell == "gru" else "g_h", "g_c"))
  m, mk = _mask_dev(d, kind)
  o = {"dgx": Buf((B, T, ng * u)), "dh0": Buf((B, u)) if opts["dh0"] else None}
  if dU:
    o["dU"] = Buf((u, ng * u))
    if cell == "gru":
      o["db_r"] = Buf((ng * u,))
  lib = _ffi.lib()
  if cell == "gru":
    ws_bytes = lib.tfrs_gru_bwd_workspace_bytes(B, T, u)
  else:
    ws_bytes = lib.tfrs_lstm_bwd_workspace_bytes(B, T, u) if dU else 0
  ws = torch.empty(max(ws_bytes, 1), dtype=torch.uint8, device="cuda")
  wsp = _p(ws) if ws_bytes else None
  pp = lambda k: o[k].p if o.get(k) is not None else None
  if cell == "gru":
    rc = lib.tfrs_gru_bwd_f32(_p(U), _p(gates), _p(h_prev), _p(m), mk, _p(g_seq), _p(g_last), B, T, u, pp("dgx"),
                              pp("dU"), pp("db_r"), pp("dh0"), wsp, ws_bytes, _ffi.stream())
  else:
    o["dc0"] = Buf((B, u)) if opts["dc0"] else None
    rc = lib.tfrs_lstm_bwd_f32(_p(U), _p(gates), _p(c_seq), _p(h_prev), _p(c0), _p(m), mk, _p(g_seq), _p(g_last),
                               _p(g_c), B, T, u, pp("dgx"), pp("dU"), pp("dh0"), pp("dc0"), wsp, ws_bytes,
                               _ffi.stream())
  _ffi.check(rc, f"{cell}_bwd")
  torch.cuda.synchronize()
  return {k: v for k, v in o.items() if v is not None}


def _bar_check(what, got, ref, err, where=None, key=None):
  """|got - ref| <= 2 u_r err per element (where given: only there); records the worst err / bar under key"""
  got = np.asarray(got, np.float64)
  sel = np.ones(ref.shape, bool) if where is None else np.broadcast_to(where, ref.shape)
  assert np.isfinite(got[sel]).all(), f"{what}: {int((~np.isfinite(got[sel])).sum())} non-finite elements"
  e = np.abs(got - ref)
  tol = re_.bar(err)
  bad = sel & (e > tol)
  if bad.any():
    i = tuple(np.argwhere(bad)[0])
    raise AssertionError(f"{what}: {int(bad.sum())} of {int(sel.sum())} elements miss the bar; first {i}: got "
                         f"{got[i]!r} ref {ref[i]!r} err {e[i]:.3e} bar {tol[i]:.3e}")
  if key is not None and sel.any():
    r = float(np.max(np.where(sel & (tol > 0), e / np.where(tol > 0, tol, 1), 0.0)))
    if r > WORST.get(key[:2], (-1, ""))[0]:
      WORST[key[:2]] = (r, key[2])


def _bits(a):
  return np.ascontiguousarray(a, np.float32).view(np.int32)


def _fp32_dh0_of_masked_row(cell, d, b, T):
  """dh0 of a fully masked row: the float32 sum from +0 in the kernel's order"""
  last = d["g_last" if cell == "gru" else "g_h"]
  s = np.zeros(d["gx"].shape[-1] // ec.NG[cell], np.float32)
  for t in reversed(range(T)):
    if d["g_seq"] is not None:
      s = s + d["g_seq"][b, t]
    if t == T - 1 and last is not None:
      s = s + last[b]
  return s


def check_forward(cell, d, kind, opts, name):
  """the forward kernel against forward_gx, with the exact masked-step, coverage and guard checks; returns the
  oracle's output (for the reverse)"""
  B, T, nu = d["gx"].shape
  u = nu // ec.NG[cell]
  keep = d["keep"]
  if cell == "gru":
    ref, err = go.forward_gx(d["gx"], d["U"], d["b_r"], d["h0"], keep)
  else:
    ref, err = lo.forward_gx(d["gx"], d["U"], d["h0"], d["c0"], keep)
  k = run_fwd(cell, d, kind, opts)
  for n, b in k.items():
    assert b.guard_ok(), f"{name}: a write past the end of {n}"
  key = (cell, "fwd", name)
  km = keep[:, :, None]
  for n in k:
    got = k[n].f32()
    if n == "gates":
      sb = k[n].bits()
      assert (sb[~keep] == SENTINEL).all(), f"{name}: gates written at a masked step"
      assert not (sb[keep] == SENTINEL).any(), f"{name}: gates of a kept step left unwritten"
      _bar_check(f"{name} gates", np.where(km, got, 0), ref[n], err[n], km, key)
    else:
      assert not (k[n].bits() == SENTINEL).any(), f"{name}: {n} not fully written"
      _bar_check(f"{name} {n}", got, ref[n], err[n], None, key)
  # exact: h_prev is h_{t-1}; out_seq at a masked step repeats it; c_seq carries; a fully masked row keeps h0 / c0
  hp = _bits(k["h_prev"].f32())
  h0 = _bits(d["h0"] if d["h0"] is not None else np.zeros((B, u), np.float32))
  assert np.array_equal(hp[:, 0], h0), f"{name}: h_prev[0] is not h0"
  assert np.array_equal(hp[:, 1:][~keep[:, :-1]], hp[:, :-1][~keep[:, :-1]]), f"{name}: h not carried"
  hT = _bits(k["h_T"].f32())
  if "seq" in k:
    sq = _bits(k["seq"].f32())
    assert np.array_equal(sq[:, :-1], hp[:, 1:]), f"{name}: h_prev[t] differs from out_seq[t-1]"
    assert np.array_equal(sq[~keep], hp[~keep]), f"{name}: out_seq at a masked step is not h_{{t-1}}"
    assert np.array_equal(sq[:, -1], hT), f"{name}: h_T differs from out_seq[T-1]"
  dead = ~keep.any(1)
  assert np.array_equal(hT[dead], h0[dead]), f"{name}: a fully masked row's h_T is not h0"
  if cell == "lstm":
    cs = _bits(k["c_seq"].f32())
    c0 = _bits(d["c0"] if d["c0"] is not None else np.zeros((B, u), np.float32))
    cprev = np.concatenate([c0[:, None], cs[:, :-1]], 1)
    assert np.array_equal(cs[~keep], cprev[~keep]), f"{name}: c not carried at a masked step"
    cT = _bits(k["c_T"].f32())
    assert np.array_equal(cT, cs[:, -1]), f"{name}: c_T differs from c_seq[T-1]"
    assert np.array_equal(cT[dead], c0[dead]), f"{name}: a fully masked row's c_T is not c0"
  return ref


def check_reverse(cell, d, kind, opts, saved, name):
  """the reverse kernel on `saved` (float32) against reverse() on the same values, with the exact checks"""
  B, T, u = saved["h_prev"].shape
  keep = d["keep"]
  if cell == "gru":
    ref, err = go.reverse(d["U"], saved["gates"], saved["h_prev"], keep, d["g_seq"], d["g_last"])
    rk = "dgx"
  else:
    ref, err = lo.reverse(d["U"], saved["gates"], saved["c_seq"], d["c0"], keep, d["g_seq"], d["g_h"], d["g_c"])
    rk = "dz"
  k = run_bwd(cell, d, saved, kind, opts)
  key = (cell, "bwd", name)
  for n, b in k.items():
    assert b.guard_ok(), f"{name}: a write past the end of {n}"
    assert not (b.bits() == SENTINEL).any(), f"{name}: {n} not fully written"
  dgx = k["dgx"].f32()
  assert (_bits(dgx)[~keep] == 0).all(), f"{name}: a masked step's gradient row is not +0"
  _bar_check(f"{name} {rk}", dgx, ref[rk], err[rk], None, key)
  dead = ~keep.any(1)
  if "dh0" in k:
    _bar_check(f"{name} dh0", k["dh0"].f32(), ref["dh0"], err["dh0"], None, key)
    for b in np.flatnonzero(dead):
      assert np.array_equal(_bits(k["dh0"].f32()[b]), _bits(_fp32_dh0_of_masked_row(cell, d, b, T))), \
          f"{name}: dh0 of fully masked row {b} is not the float32 sum of its upstream gradients"
  if "dc0" in k:
    _bar_check(f"{name} dc0", k["dc0"].f32(), ref["dc0"], err["dc0"], None, key)
    gc = d["g_c"] if d["g_c"] is not None else np.zeros((B, u), np.float32)
    exp = np.float32(0) + gc
    assert np.array_equal(_bits(k["dc0"].f32()[dead]), _bits(exp[dead])), f"{name}: a fully masked row's dc0 is not g_c"
  return k


def _saved32(cell, ref):
  names = ("gates", "h_prev") + (("c_seq",) if cell == "lstm" else ())
  return {n: ref[n].astype(np.float32) for n in names}


def check_both(cell, d, kind, opts, name):
  ref = check_forward(cell, d, kind, opts, name)
  check_reverse(cell, d, kind, opts, _saved32(cell, ref), name)


@pytest.mark.parametrize("case", ec.CASES, ids=[c.name for c in ec.CASES])
def test_case_matches_the_oracle_per_element(case):
  d = ec.inputs(case)
  check_both(case.cell, d, case.kind, ec.OPTS[case.cell][case.opts], case.name)


# ---- row isolation -----------------------------------------------------------------------------------------------------
ISO = [(cell, uj, kind) for cell in ec.CELLS for uj in ec.UJS for kind in ec.MASK_KINDS]


@pytest.mark.parametrize("cell,uj,kind", ISO, ids=[f"{c}-uj{j}-{k}" for c, j, k in ISO])
def test_a_rows_nan_and_inf_stay_in_that_row(cell, uj, kind):
  """NaN / Inf in one row's gx, h0, c0 and upstream gradients, that row first in a CTA, last in a CTA and in the final
  partial CTA: every other row's outputs and gradients keep their bits."""
  u = ec.REP_U[uj] + 7
  R = ec.tile(u).rows
  B = 2 * R + max(1, R // 2)
  case = ec.Case(f"iso-{cell}-{uj}-{kind}", cell, u, B, 3, kind, "random", 0, 77 + uj)
  opts = ec.OPTS[cell][0]
  clean = ec.inputs(case)
  bad = {k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in clean.items()}
  rows = sorted({R, 2 * R - 1, B - 1})
  for b in rows:
    bad["gx"][b, 0, ::2] = np.nan
    bad["gx"][b, -1, 1::2] = np.inf
    bad["h0"][b] = np.nan
    if cell == "lstm":
      bad["c0"][b] = -np.inf
    bad["g_seq"][b, 1] = np.nan
    bad["g_last" if cell == "gru" else "g_h"][b] = np.inf
    if cell == "lstm":
      bad["g_c"][b] = np.nan
  others = np.setdiff1d(np.arange(B), rows)
  outs = []
  for d in (clean, bad):
    f = run_fwd(cell, d, kind, opts)
    saved = {n: f[n].f32() for n in ("gates", "h_prev", "c_seq") if n in f}
    r = run_bwd(cell, d, saved, kind, opts)
    outs.append({**{n: b.bits() for n, b in f.items() if n != "gates"}, **{n: b.bits() for n, b in r.items()},
                 "gates": f["gates"].bits()})
  for n in outs[0]:
    assert np.array_equal(outs[0][n][others], outs[1][n][others]), f"{n}: a poisoned row changed another row"
  assert not np.isfinite(outs[1]["h_T"][rows].view(np.float32)).all()


# ---- saturation --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cell", ec.CELLS)
@pytest.mark.parametrize("u", [33, 300])
def test_saturated_gates(cell, u):
  """Pre-activations of +-20 to +-90 (|c| large enough that tanhf saturates for LSTM): the saved sigmoid / tanh outputs
  are exactly 0 or +-1, and the derivatives the reverse takes from them are exactly 0 where they are."""
  case = ec.Case(f"sat-{cell}-{u}", cell, u, ec.tile(u).rows + 1, 5, "bool", "random", 0, 300 + u)
  d = ec.inputs(case)
  rng = np.random.RandomState(u)
  mag = rng.uniform(20, 90, size=d["gx"].shape)
  d["gx"] = (np.where(rng.rand(*mag.shape) < 0.5, -mag, mag)).astype(np.float32)
  if cell == "lstm":
    d["c0"] = (rng.choice([-1, 1], size=d["c0"].shape) * rng.uniform(20, 60, size=d["c0"].shape)).astype(np.float32)
  opts = ec.OPTS[cell][0]
  ref = check_forward(cell, d, case.kind, opts, case.name)
  saved = _saved32(cell, ref)
  g = saved["gates"]
  k = check_reverse(cell, d, case.kind, opts, saved, case.name)
  dgx = k["dgx"].f32()
  keep = d["keep"][:, :, None]
  sat = lambda s: (s == 0) | (s == 1)
  if cell == "gru":
    z, r, hh = g[..., :u], g[..., u:2 * u], g[..., 2 * u:3 * u]
    dead_dhp = (z == 1) | (np.abs(hh) == 1)
    zero = {0: sat(z), 1: sat(r) | dead_dhp, 2: dead_dhp}
  else:
    i, f, gg, o = (g[..., q * u:(q + 1) * u] for q in range(4))
    zero = {0: sat(i), 1: sat(f), 2: np.abs(gg) == 1, 3: sat(o)}
  for q, z0 in zero.items():
    sel = z0 & keep
    assert sel.mean() > 0.2, f"gate block {q} did not saturate"
    assert (dgx[..., q * u:(q + 1) * u][sel] == 0).all(), f"gate block {q}: a saturated gate's gradient is not 0"


# ---- dU and db_r through the C entry's K6 call --------------------------------------------------------------------------
def _ebar(A, B):
  """tests/test_gpu_split_gemm_edges.py's per-element bar (E) for A . B"""
  Af, Bf = np.abs(A), np.abs(B)
  return 1e-5 * (Af @ Bf) + 2.0 ** -36 * (Af.max() * Bf.sum(0)[None, :] + Bf.max() * Af.sum(1)[:, None])


@pytest.mark.parametrize("cell", ec.CELLS)
@pytest.mark.parametrize("u,B,T", [(33, 40, 7), (300, 70, 5)])
def test_dU_and_db_r_through_the_entry_point(cell, u, B, T):
  """dU = h_prev^T . dgr (and GRU's db_r = colsum(dgr)) from the kernel's own gradient rows: GRU's dgr is dgx with the
  last block times r, one float32 multiply"""
  case = ec.Case(f"dU-{cell}-{u}", cell, u, B, T, "int64", "edges", 0, 500 + u)
  d = ec.inputs(case)
  opts = ec.OPTS[cell][0]
  ref = check_forward(cell, d, case.kind, opts, case.name)
  saved = _saved32(cell, ref)
  k = run_bwd(cell, d, saved, case.kind, opts, dU=True)
  for n, b in k.items():
    assert b.guard_ok() and not (b.bits() == SENTINEL).any(), n
  ng = ec.NG[cell]
  dg = k["dgx"].f32().reshape(B * T, ng * u).copy()
  keep = d["keep"].reshape(B * T)
  if cell == "gru":
    r = saved["gates"].reshape(B * T, 4 * u)[:, u:2 * u]
    dg[:, 2 * u:] = np.where(keep[:, None], dg[:, 2 * u:] * r, 0).astype(np.float32)
  A = saved["h_prev"].reshape(B * T, u).T.astype(np.float64)
  dg = dg.astype(np.float64)
  _bar_check_abs("dU", k["dU"].f32(), A @ dg, _ebar(A, dg))
  if cell == "gru":
    ones = np.ones((1, B * T))
    _bar_check_abs("db_r", k["db_r"].f32()[None], ones @ dg, _ebar(ones, dg))


def _bar_check_abs(what, got, ref, tol):
  got = np.asarray(got, np.float64)
  assert np.isfinite(got).all(), what
  e = np.abs(got - ref)
  assert (e <= tol).all(), f"{what}: max err / bar {float((e / tol).max()):.3g}"


# ---- gates / dgx offsets past 2^31 elements ----------------------------------------------------------------------------
def test_offsets_past_two_to_the_31():
  """GRU at u = 256, B = 16387, T = 129: gates hold B T 4u > 2^31 elements and dgx B T 3u > 2^31 - 2^30.  The first row,
  the row holding gates element 2^31 and the last row meet the oracle, the reverse fed the forward's own saves."""
  u, B, T = 256, 16387, 129
  assert B * T * 4 * u > 2 ** 31
  lib = _ffi.lib()
  ws_bytes = lib.tfrs_gru_bwd_workspace_bytes(B, T, u)
  # the reverse's peak: gates, h_prev, g_seq, dgx and the workspace (gx is freed after the forward)
  need = B * T * u * 4 * (4 + 1 + 1 + 3) + ws_bytes + (1 << 30)
  free = torch.cuda.mem_get_info()[0]
  if free < need:
    pytest.skip(f"needs {need / 2 ** 30:.1f} GiB of free device memory, {free / 2 ** 30:.1f} GiB free")
  cell = "gru"
  rows = [0, 2 ** 31 // (T * 4 * u), B - 1]
  case = ec.Case("big", cell, u, B, T, None, "random", 0, 9)
  opts = dict(h0=1, br=1, seq=0, g_seq=1, g_last=1, dh0=1)
  small = ec.inputs(ec.Case("big", cell, u, len(rows), T, None, "random", 0, 9))
  gen = torch.Generator(device="cuda").manual_seed(5)
  d = {"U": small["U"], "b_r": small["b_r"], "keep": np.ones((B, T), bool), "mask": None,
       "gx": None, "h0": None, "g_seq": None, "g_last": None}
  gx = torch.randn((B, T, 3 * u), device="cuda", generator=gen)
  h0 = torch.rand((B, u), device="cuda", generator=gen) - 0.5
  U, br = _dev(d["U"]), _dev(d["b_r"])
  hT, gates, hprev = Buf((B, u)), Buf((B, T, 4 * u)), Buf((B, T, u))
  _ffi.check(lib.tfrs_gru_fwd_f32(_p(gx), _p(U), _p(br), _p(h0), None, 0, B, T, u, None, hT.p,
                                  gates.p, hprev.p, _ffi.stream()), "gru_fwd")
  torch.cuda.synchronize()
  gx_rows = gx[rows].cpu().numpy()
  del gx
  for b in (hT, gates, hprev):
    assert b.guard_ok() and not bool((b.raw[:b.n] == SENTINEL).any())
  ref, err = go.forward_gx(gx_rows, d["U"], d["b_r"], h0[rows].cpu().numpy(), None)
  sl = lambda b: b.raw[:b.n].view(b.shape)[rows].cpu().numpy().view(np.float32)
  for n, b in (("h_T", hT), ("gates", gates), ("h_prev", hprev)):
    _bar_check(f"big {n}", sl(b), ref[n], err[n])
  g_seq = torch.randn((B, T, u), device="cuda", generator=gen)
  g_last = torch.randn((B, u), device="cuda", generator=gen)
  dgx, dh0 = Buf((B, T, 3 * u)), Buf((B, u))
  ws = torch.empty(ws_bytes, dtype=torch.uint8, device="cuda")
  gv, hv = gates.raw[:gates.n].view(torch.float32), hprev.raw[:hprev.n].view(torch.float32)
  _ffi.check(lib.tfrs_gru_bwd_f32(_p(U), _p(gv), _p(hv), None, 0, _p(g_seq), _p(g_last), B, T, u, dgx.p,
                                  None, None, dh0.p, _p(ws), ws_bytes, _ffi.stream()), "gru_bwd")
  torch.cuda.synchronize()
  del ws
  for b in (dgx, dh0):
    assert b.guard_ok() and not bool((b.raw[:b.n] == SENTINEL).any())
  rr, re = go.reverse(d["U"], sl(gates), sl(hprev), None, g_seq[rows].cpu().numpy(), g_last[rows].cpu().numpy())
  _bar_check("big dgx", sl(dgx), rr["dgx"], re["dgx"])
  _bar_check("big dh0", sl(dh0), rr["dh0"], re["dh0"])
