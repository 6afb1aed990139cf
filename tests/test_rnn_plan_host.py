"""CPU checks of the K19 / K20 recurrence edge cases and bars (tests/rnn_edge_cases.py, tests/rnn_error.py, the
forward_gx / reverse oracles):
  - the plan constants are csrc/rnn.cuh's, and the generated cases reach every instance, resident / streamed flip, slice
    edge, batch and length edge, mask kind, pattern and mask value, so a changed constant fails here instead of silently
    dropping coverage;
  - the bars accept a float32 NumPy evaluation of the header's formulas in the kernels' operation order;
  - the bars, loosened 16x, still reject float64 mutants of the recurrence;
  - the bars are not vacuous: the median bar / |value| of every output of every case is below 2^-12 (dh0, the U^T
    chain alone: 2^-12 NG u / 1024 beyond NG u = 1024)."""
import os
import re

import numpy as np
import pytest

import gru_oracle as go
import lstm_oracle as lo
import rnn_edge_cases as ec
import rnn_error as re_

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HOST_ROWS = 4            # rows are independent: the host checks run a case on its first rows


def _header_const(name):
  src = open(os.path.join(ROOT, "recommenders_b200", "csrc", "rnn.cuh")).read()
  m = re.search(r"constexpr int %s = ([0-9 *]+);" % name, src)
  assert m, name
  return eval(m.group(1))


def test_the_plan_constants_are_the_headers():
  assert (_header_const("RNN_THREADS"), _header_const("RNN_PAIRS"), _header_const("RNN_SMEM_MAX"),
          _header_const("RNN_SLICE_BYTES")) == (ec.THREADS, ec.PAIRS, ec.SMEM_MAX, ec.SLICE_BYTES)
  hdr = open(os.path.join(ROOT, "include", "tfrs_b200.h")).read()
  for n in ("GRU", "LSTM"):
    assert int(re.search(r"#define TFRS_%s_MAX_UNITS (\d+)" % n, hdr).group(1)) == ec.MAX_UNITS


def test_the_plan_matches_the_documented_flips():
  assert ec.resident_edges("gru", "fwd") == [136] and ec.resident_edges("gru", "bwd") == [123, 128, 130]
  assert ec.resident_edges("lstm", "fwd") == [116] and ec.resident_edges("lstm", "bwd") == [105]
  assert [ec.tile(u).uj for u in (256, 257, 512, 513, 1024, 1025, 2048)] == [1, 2, 2, 4, 4, 8, 8]


def _coverage():
  """the per-instance coverage table: (cell, direction, UJ) -> what the cases reach there"""
  t = {}
  for c in ec.CASES:
    for d in ec.DIRS:
      p = ec.plan(c.cell, d, c.u)
      e = t.setdefault((c.cell, d, p.tile.uj), {"kinds": set(), "resident": set(), "last": set(), "exact": False})
      e["kinds"].add(c.kind)
      e["resident"].add(p.resident)
      if not p.resident:
        e["last"].add(p.last)
        e["exact"] |= p.last == p.slice_rows
  return t


def test_the_cases_reach_every_instance_and_slice_edge():
  t = _coverage()
  for cell in ec.CELLS:
    for d in ec.DIRS:
      for uj in ec.UJS:
        e = t[(cell, d, uj)]
        assert e["kinds"] == set(ec.MASK_KINDS), (cell, d, uj)
        assert False in e["resident"], (cell, d, uj)
        assert True in e["resident"] or uj > 1, (cell, d, uj)
        shortest = min(ec.plan(cell, d, u).last for u in ec.units_of(uj) if not ec.plan(cell, d, u).resident)
        assert shortest in e["last"] and e["exact"], (cell, d, uj)
        assert shortest == 1 or (cell, d, uj) == ("lstm", "bwd", 1), (cell, d, uj, shortest)
      for edge in ec.resident_edges(cell, d):
        assert {edge, edge + 1} <= {c.u for c in ec.CASES if c.cell == cell}, (cell, d, edge)
  print("\n(cell, dir, UJ): mask kinds / resident and streamed / last-slice sizes reached")
  for k, e in sorted(t.items()):
    print(k, sorted(map(str, e["kinds"])), sorted(e["resident"]), sorted(e["last"]), "exact" if e["exact"] else "")


def test_the_cases_reach_every_batch_length_pattern_and_mask_value():
  for cell in ec.CELLS:
    cs = [c for c in ec.CASES if c.cell == cell]
    for u in (33, 257):
      R = ec.tile(u).rows
      assert {1, R - 1, R, R + 1} <= {c.B for c in cs if c.u == u}
    assert any(-(-c.B // ec.tile(c.u).rows) > ec.WAVE_CTAS for c in cs)
    Ts = {c.T for c in cs}
    assert {1, 2, 3} <= Ts and any(T >= 65 and T % 2 for T in Ts) and any(T >= 999 for T in Ts)
    assert any(c.T >= 999 and c.contractive and c.kind for c in cs)
    assert {c.pattern for c in cs if c.kind} == set(ec.PATTERNS)
    assert {c.opts for c in cs} == set(range(len(ec.OPTS[cell])))
    for kind in ("int32", "int64"):
      seen = set()
      for c in cs:
        if c.kind == kind:
          m = ec.inputs(c)["mask"]
          seen |= set(np.unique(m).tolist())
      assert set(ec.NONZERO[kind]) | {0} <= seen, (cell, kind, seen)
    edges = [c for c in cs if c.pattern == "edges" and c.kind and c.B >= 3 and c.T >= 2]
    assert edges
    k = ec.inputs(edges[0])["keep"]
    assert not k[0].any() and not k[1, 0] and k[1, 1:].all() and not k[2, -1] and k[2, :-1].all()


def test_the_gpu_cases_pass_the_mask_values_not_just_keep():
  c = next(c for c in ec.CASES if c.kind == "int64" and c.B > 1)
  d = ec.inputs(c)
  assert d["mask"].dtype == np.int64 and np.array_equal(d["mask"] != 0, d["keep"])
  assert (d["mask"] == 2 ** 32).any() or (d["mask"] == ec.INT64_MIN).any()


# ---- the float32 evaluation the bars must accept -------------------------------------------------------------------------
f32 = np.float32


def _chain32(x, W):
  """fmaf over k ascending from +0: each step exact in float64 (a 24 x 24-bit product and one add of it), rounded"""
  acc = np.zeros((x.shape[0], W.shape[1]), f32)
  for k in range(x.shape[1]):
    acc = (acc.astype(np.float64) + x[:, k:k + 1].astype(np.float64) * W[k].astype(np.float64)).astype(f32)
  return acc


def _sig32(x):
  with np.errstate(over="ignore"):
    return f32(1) / (f32(1) + np.exp(-x))


def gru_fwd32(d):
  gx, U, br = d["gx"], d["U"], d["b_r"]
  B, T, _ = gx.shape
  u = U.shape[0]
  h = d["h0"].copy() if d["h0"] is not None else np.zeros((B, u), f32)
  seq, gates, hprev = np.zeros((B, T, u), f32), np.zeros((B, T, 4 * u), f32), np.zeros((B, T, u), f32)
  for t in range(T):
    a = _chain32(h, U)
    if br is not None:
      a = a + br
    z = _sig32(gx[:, t, :u] + a[:, :u])
    r = _sig32(gx[:, t, u:2 * u] + a[:, u:2 * u])
    hh = np.tanh(gx[:, t, 2 * u:] + r * a[:, 2 * u:])
    hn = z * h + (f32(1) - z) * hh
    gates[:, t] = np.concatenate([z, r, hh, a[:, 2 * u:]], 1)
    hprev[:, t] = h
    h = np.where(d["keep"][:, t:t + 1], hn, h)
    seq[:, t] = h
  return {"seq": seq, "h_T": h, "gates": gates, "h_prev": hprev}


def lstm_fwd32(d):
  gx, U = d["gx"], d["U"]
  B, T, _ = gx.shape
  u = U.shape[0]
  h = d["h0"].copy() if d["h0"] is not None else np.zeros((B, u), f32)
  c = d["c0"].copy() if d["c0"] is not None else np.zeros((B, u), f32)
  out = {n: np.zeros((B, T, m * u), f32) for n, m in (("seq", 1), ("gates", 4), ("c_seq", 1), ("h_prev", 1))}
  for t in range(T):
    z = gx[:, t] + _chain32(h, U)
    i, f, g, o = _sig32(z[:, :u]), _sig32(z[:, u:2 * u]), np.tanh(z[:, 2 * u:3 * u]), _sig32(z[:, 3 * u:])
    cn = f * c + i * g
    hn = o * np.tanh(cn)
    out["gates"][:, t] = np.concatenate([i, f, g, o], 1)
    out["h_prev"][:, t] = h
    k = d["keep"][:, t:t + 1]
    h, c = np.where(k, hn, h), np.where(k, cn, c)
    out["seq"][:, t], out["c_seq"][:, t] = h, c
  out["h_T"], out["c_T"] = h, c
  return out


def gru_rev32(d, s):
  U, gates, hprev = d["U"], s["gates"], s["h_prev"]
  B, T, u = hprev.shape
  dh = np.zeros((B, u), f32)
  dgx = np.zeros((B, T, 3 * u), f32)
  for t in reversed(range(T)):
    dd = dh
    if d["g_seq"] is not None:
      dd = dd + d["g_seq"][:, t]
    if d["g_last"] is not None and t == T - 1:
      dd = dd + d["g_last"]
    g = gates[:, t]
    z, r, hh, grh = g[:, :u], g[:, u:2 * u], g[:, 2 * u:3 * u], g[:, 3 * u:]
    dz = dd * (hprev[:, t] - hh) * (z * (f32(1) - z))
    dhp = dd * (f32(1) - z) * (f32(1) - hh * hh)
    dr = dhp * grh * (r * (f32(1) - r))
    k = d["keep"][:, t:t + 1]
    dgr = np.where(k, np.concatenate([dz, dr, dhp * r], 1), f32(0))
    dgx[:, t] = np.where(k, np.concatenate([dz, dr, dhp], 1), f32(0))
    dh = np.where(k, dd * z + _chain32(dgr, U.T), dd)
  return {"dgx": dgx, "dh0": dh}


def lstm_rev32(d, s):
  U, gates, cs = d["U"], s["gates"], s["c_seq"]
  B, T, u = cs.shape
  c0 = d["c0"] if d["c0"] is not None else np.zeros((B, u), f32)
  dh, dc = np.zeros((B, u), f32), np.zeros((B, u), f32)
  dz = np.zeros((B, T, 4 * u), f32)
  for t in reversed(range(T)):
    dd = dh
    if d["g_seq"] is not None:
      dd = dd + d["g_seq"][:, t]
    if t == T - 1:
      if d["g_h"] is not None:
        dd = dd + d["g_h"]
      if d["g_c"] is not None:
        dc = dc + d["g_c"]
    g = gates[:, t]
    i, f, gg, o = g[:, :u], g[:, u:2 * u], g[:, 2 * u:3 * u], g[:, 3 * u:]
    cp = cs[:, t - 1] if t > 0 else c0
    tc = np.tanh(cs[:, t])
    do = dd * tc * (o * (f32(1) - o))
    dct = dc + dd * o * (f32(1) - tc * tc)
    k = d["keep"][:, t:t + 1]
    z = np.where(k, np.concatenate([dct * gg * (i * (f32(1) - i)), dct * cp * (f * (f32(1) - f)),
                                    dct * i * (f32(1) - gg * gg), do], 1), f32(0))
    dz[:, t] = z
    dh = np.where(k, _chain32(z, U.T), dd)
    dc = np.where(k, dct * f, dc)
  return {"dz": dz, "dh0": dh, "dc0": dc}


def _oracle(cell, d):
  if cell == "gru":
    ref, err = go.forward_gx(d["gx"], d["U"], d["b_r"], d["h0"], d["keep"])
  else:
    ref, err = lo.forward_gx(d["gx"], d["U"], d["h0"], d["c0"], d["keep"])
  names = ("gates", "h_prev") + (("c_seq",) if cell == "lstm" else ())
  saved = {n: ref[n].astype(f32) for n in names}
  if cell == "gru":
    rr, rerr = go.reverse(d["U"], saved["gates"], saved["h_prev"], d["keep"], d["g_seq"], d["g_last"])
  else:
    rr, rerr = lo.reverse(d["U"], saved["gates"], saved["c_seq"], d["c0"], d["keep"], d["g_seq"], d["g_h"], d["g_c"])
  return ref, err, saved, rr, rerr


def _ratio(got, ref, err, keep=None):
  """max |got - ref| / bar, over kept steps for gates"""
  e = np.abs(np.asarray(got, np.float64) - ref)
  tol = re_.bar(err)
  if keep is not None:
    e = e * keep[:, :, None]
  with np.errstate(divide="ignore", invalid="ignore"):
    r = np.where(e == 0, 0.0, e / tol)
  return float(np.nan_to_num(r, nan=np.inf).max()) if r.size else 0.0


def _small(case):
  return case.u <= 140 and case.T <= 129


SMALL = [c for c in ec.CASES if _small(c)]


@pytest.mark.parametrize("case", SMALL, ids=[c.name for c in SMALL])
def test_the_bars_accept_the_float32_formulas(case):
  d = ec.inputs(case, rows=np.arange(min(case.B, HOST_ROWS)))
  ref, err, saved, rr, rerr = _oracle(case.cell, d)
  fwd = gru_fwd32(d) if case.cell == "gru" else lstm_fwd32(d)
  for n, v in fwd.items():
    assert _ratio(v, ref[n], err[n], d["keep"] if n == "gates" else None) <= 1, n
  rev = gru_rev32(d, saved) if case.cell == "gru" else lstm_rev32(d, saved)
  for n, v in rev.items():
    assert _ratio(v, rr[n], rerr[n]) <= 1, n


@pytest.mark.parametrize("case", ec.CASES, ids=[c.name for c in ec.CASES])
def test_the_bars_are_not_vacuous(case):
  d = ec.inputs(case, rows=np.arange(min(case.B, HOST_ROWS)))
  ref, err, _, rr, rerr = _oracle(case.cell, d)
  for n in err:
    v, e = np.abs(ref[n]), re_.bar(err[n])
    if n == "gates":
      v, e = v[d["keep"]], e[d["keep"]]
    sel = v > 0
    if sel.any():
      assert np.median(e[sel] / v[sel]) < 2.0 ** -12, (n, np.median(e[sel] / v[sel]))
  for n in rerr:
    v, e = np.abs(rr[n]), re_.bar(rerr[n])
    sel = v > 0
    # dh0 of a kept step 0 is the U^T chain alone, a cancelling sum of NG u products: a worst-case bound of it grows
    # about linearly in the length where its value grows like the square root
    lim = 2.0 ** -12 * (max(1.0, ec.NG[case.cell] * case.u / 1024) if n == "dh0" else 1.0)
    if sel.any():
      assert np.median(e[sel] / v[sel]) < lim, (n, np.median(e[sel] / v[sel]))


# ---- float64 mutants the bars must reject, loosened 16x ------------------------------------------------------------------
def _gru_fwd_mutant(d, reset_before=False, drop_last=0, swap_z=False, late_mask=False):
  gx, U = d["gx"].astype(np.float64), d["U"].astype(np.float64)
  br = np.zeros(U.shape[1]) if d["b_r"] is None else d["b_r"].astype(np.float64)
  B, T, _ = gx.shape
  u = U.shape[0]
  h = d["h0"].astype(np.float64) if d["h0"] is not None else np.zeros((B, u))
  keep = d["keep"]
  if late_mask:
    keep = np.concatenate([np.ones((B, 1), bool), keep[:, :-1]], 1)
  seq = np.zeros((B, T, u))
  n = u - drop_last
  for t in range(T):
    a = h[:, :n] @ U[:n] + br
    z = go.sigmoid(gx[:, t, :u] + a[:, :u])
    r = go.sigmoid(gx[:, t, u:2 * u] + a[:, u:2 * u])
    if reset_before:
      hh = np.tanh(gx[:, t, 2 * u:] + (r * h) @ U[:, 2 * u:] + br[2 * u:])
    else:
      hh = np.tanh(gx[:, t, 2 * u:] + r * a[:, 2 * u:])
    hn = (1 - z) * h + z * hh if swap_z else z * h + (1 - z) * hh
    h = np.where(keep[:, t:t + 1], hn, h)
    seq[:, t] = h
  return {"seq": seq, "h_T": h}


def _lstm_fwd_mutant(d, drop_last=0, late_mask=False):
  gx, U = d["gx"].astype(np.float64), d["U"].astype(np.float64)
  B, T, _ = gx.shape
  u = U.shape[0]
  h = d["h0"].astype(np.float64) if d["h0"] is not None else np.zeros((B, u))
  c = d["c0"].astype(np.float64) if d["c0"] is not None else np.zeros((B, u))
  keep = d["keep"]
  if late_mask:
    keep = np.concatenate([np.ones((B, 1), bool), keep[:, :-1]], 1)
  seq = np.zeros((B, T, u))
  n = u - drop_last
  for t in range(T):
    z = gx[:, t] + h[:, :n] @ U[:n]
    i, f, g, o = lo.sigmoid(z[:, :u]), lo.sigmoid(z[:, u:2 * u]), np.tanh(z[:, 2 * u:3 * u]), lo.sigmoid(z[:, 3 * u:])
    cn = f * c + i * g
    k = keep[:, t:t + 1]
    h, c = np.where(k, o * np.tanh(cn), h), np.where(k, cn, c)
    seq[:, t] = h
  return {"seq": seq, "h_T": h, "c_T": c}


def _lstm_rev_mutant(d, s, wrong_cp=False, dc_dropped=False):
  U, gates, cs = d["U"].astype(np.float64), s["gates"].astype(np.float64), s["c_seq"].astype(np.float64)
  B, T, u = cs.shape
  c0 = d["c0"].astype(np.float64) if d["c0"] is not None else np.zeros((B, u))
  keep = d["keep"]
  cprev = np.concatenate([c0[:, None], cs[:, :-1]], 1)     # c_{t-1}
  if wrong_cp:
    # c_{t-1} of the previous kept step: after a masked step the c from before the step before it
    for b in range(B):
      last = None
      for t in range(T):
        if keep[b, t]:
          if last is not None and last != t - 1:
            cprev[b, t] = c0[b] if last == 0 else cs[b, last - 1]
          last = t
  dh, dc = np.zeros((B, u)), np.zeros((B, u))
  dz = np.zeros((B, T, 4 * u))
  for t in reversed(range(T)):
    dd = dh + (d["g_seq"][:, t] if d["g_seq"] is not None else 0)
    if t == T - 1:
      dd = dd + (d["g_h"] if d["g_h"] is not None else 0)
      dc = dc + (d["g_c"] if d["g_c"] is not None else 0)
    g = gates[:, t]
    i, f, gg, o = g[:, :u], g[:, u:2 * u], g[:, 2 * u:3 * u], g[:, 3 * u:]
    tc = np.tanh(cs[:, t])
    dct = dc + dd * o * (1 - tc * tc)
    k = keep[:, t:t + 1]
    z = np.concatenate([dct * gg * i * (1 - i), dct * cprev[:, t] * f * (1 - f), dct * i * (1 - gg * gg),
                        dd * tc * o * (1 - o)], 1) * k
    dz[:, t] = z
    dh = np.where(k, z @ U.T, dd)
    dc = np.where(k, dct * f, 0.0 if dc_dropped else dc)
  return {"dz": dz, "dh0": dh, "dc0": dc}


def _mutant_case(cell, u, pattern, T=6, B=6, opts=0, seed=5):
  return ec.Case(f"mutant-{cell}", cell, u, B, T, "bool", pattern, opts, seed)


MUTANTS = {
    "gru reset gate before h.U (reset_after=False)": ("gru", 33, "random", dict(reset_before=True)),
    "gru last U slice dropped": ("gru", 181, "random", "drop"),
    "gru z and 1 - z swapped": ("gru", 33, "random", dict(swap_z=True)),
    "gru mask one step late": ("gru", 33, "edges", dict(late_mask=True)),
    "lstm last U slice dropped": ("lstm", 157, "random", "drop"),
    "lstm mask one step late": ("lstm", 33, "edges", dict(late_mask=True)),
    "lstm c_{t-1} from the wrong step after a masked step": ("lstm", 33, "random", dict(wrong_cp=True)),
    "lstm dc not passed through a masked step": ("lstm", 33, "random", dict(dc_dropped=True)),
}


@pytest.mark.parametrize("what", sorted(MUTANTS))
def test_the_bars_reject_mutants_with_16x_margin(what):
  cell, u, pattern, kw = MUTANTS[what]
  case = _mutant_case(cell, u, pattern)
  d = ec.inputs(case)
  ref, err, saved, rr, rerr = _oracle(cell, d)
  if kw == "drop":
    p = ec.plan(cell, "fwd", u)
    assert not p.resident and p.last == 1
    kw = dict(drop_last=p.last)
  if "wrong_cp" in kw or "dc_dropped" in kw:
    got = _lstm_rev_mutant(d, saved, **kw)
    r = max(_ratio(got[n], rr[n], rerr[n]) for n in got)
    # the float64 reference itself passes
    assert max(_ratio(v, rr[n], rerr[n]) for n, v in _lstm_rev_mutant(d, saved).items()) <= 1
  else:
    got = _gru_fwd_mutant(d, **kw) if cell == "gru" else _lstm_fwd_mutant(d, **kw)
    r = max(_ratio(got[n], ref[n], err[n]) for n in got)
  assert r > 16, f"{what}: max err / bar only {r:.3g}"
