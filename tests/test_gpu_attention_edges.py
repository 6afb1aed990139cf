"""K21 and K25 (csrc/attention.cuh) on the H100, kernel by kernel, every output and gradient held per element against
the float64 oracles (tests/attention_oracle.py, tests/dense_attention_oracle.py) at the shapes
tests/attention_edge_cases.py derives from the staged-tile plan: every head-width instance E, the tile - 1 / tile /
tile + 1 / two / three-tile walks of each width (down to the 1- and 2-row tiles of dk = dv = 128), CTAs packed with up
to 32 sequences and ending in dead teams, online-softmax scores spanning +-80 (ascending, descending, equal, one
dominant key, fully masked rows), the returned P, sequence isolation, and the dense modes' dropout, causal masks and
weight gradients at the same edges.

The bars.  Each element must lie within 2 u B of the oracle, u = 2^-24, where B is the largest first-order error bound
of the element's row ((b, h, t) for O, P and dQ; (b, h, s) for dK and dV) that core_error_bounds / error_bounds derive
from the kernels' fp32 operation counts: the score's fmaf chain over the head dims (ceil(d / 8) per lane, 3 butterfly
adds) times the magnitude sum_d |q_d k_d| of its terms, the softmax's S-term sums and rescales, expf and __fdividef,
and the T- or S-term fmaf chains of the gradients.  The factor 2 covers the second-order terms those bounds drop; a
row whose bound is 0 (an output-masked row) must be exact.  The scalar weight gradients sum B * Tq rows whose
contributions cancel, so they keep tests/test_gpu_dense_attention.py's 1e-5 row-sum bar, with each row's ds_j =
w_j (dw_j - delta) counted at its uncancelled size w_j (|dw_j| + |delta|) (dense_attention_oracle.
weight_grad_magnitudes): fp32 forms ds from that difference, which at Tv = 1 cancels to exactly 0 in float64 but to a
rounding residue in fp32.  The additive dscale is held so per column."""
import numpy as np
import pytest
import torch

import attention_edge_cases as cases
import attention_oracle as ao
import dense_attention_oracle as dao
import regularization_oracle as ro
from recommenders_b200 import ops

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
SLACK = 2.0


def _cu(a, grad=False):
  return None if a is None else torch.from_numpy(np.ascontiguousarray(a)).cuda().requires_grad_(grad)


def _np(t):
  return t.detach().double().cpu().numpy()


def _bits_equal(a, b):
  """bitwise equality, NaN payloads included"""
  return torch.equal(a.detach().contiguous().view(torch.int32), b.detach().contiguous().view(torch.int32))


def _rows(name, got, exp, bound):
  """|got - exp| <= SLACK u max(bound over the last axis), element by element."""
  got = _np(got).reshape(exp.shape)
  bar = SLACK * U * bound.max(-1, keepdims=True)
  err = np.abs(got - exp)
  bad = ~(err <= bar)
  if bad.any():
    i = np.unravel_index(np.argmax(np.where(bad, err / np.maximum(bar, 1e-300), -1.0)), exp.shape)
    raise AssertionError(f"{name}: {int(bad.sum())} of {exp.size} elements over their row's bar; worst at {i}: got "
                         f"{got[i]!r}, oracle {exp[i]!r}, bar {float(np.broadcast_to(bar, exp.shape)[i]):.3g}")


# ---- A. the MHA core through ops.attention_core --------------------------------------------------------------------
def _spread(x):
  """x in [-1, 1] -> scores in [-80, -34] u [-30, 30] u [34, 80], increasing: no score within 2 of +-32, where
  s + (-1e9) changes its fp32 rounding (the multiples of 64), so a masked score rounds as the oracle's cast does."""
  p = (np.asarray(x, np.float64) + 1) / 2 * 152
  return np.where(p < 46, -80 + p, np.where(p < 106, p - 76, p - 72))


def _core_inputs(B, T, S, H, dk, dv, seed):
  """Q, K, V [B, L, H, d] and dO with sequence n = b H + h's scores s_ts ~ beta_s of pattern n % 5: ascending along S
  (the max grows at every key), descending, all equal (identical key rows), one dominant key at 80 over [-5, 5], and
  spread.  The beta sits in the last head dim; the others carry noise of about 0.05 in the score."""
  rng = np.random.RandomState(seed)
  Q = rng.normal(size=(B, T, H, dk))
  K = rng.normal(size=(B, S, H, dk)) * 0.05
  Q[..., -1] = np.float32(1.0 / ao.scale_of(dk))
  for n in range(B * H):
    b, h = divmod(n, H)
    kind = n % 5
    if kind == 0:
      beta = _spread(np.linspace(-1, 1, S))
    elif kind == 1:
      beta = _spread(np.linspace(1, -1, S))
    elif kind == 2:
      K[b, :, h] = K[b, 0, h]
      beta = np.full(S, 50.0)
    elif kind == 3:
      beta = rng.uniform(-5, 5, S)
      beta[rng.randint(S)] = 80.0
    else:
      beta = _spread(rng.uniform(-1, 1, S))
    K[b, :, h, -1] = beta
  V = rng.normal(size=(B, S, H, dv))
  dO = rng.normal(size=(B, T, H, dv))
  return [a.astype(np.float32) for a in (Q, K, V, dO)]


def _core_call(Q, K, V, dO, H, qm, causal):
  """(O [B,T,H,dv], P [B,H,T,S], dQ, dK, dV) from the kernels, with P checked bitwise against a no-grad call."""
  B, T, S = Q.shape[0], Q.shape[1], K.shape[1]
  tq, tk, tv = (_cu(a.reshape(a.shape[0], a.shape[1], -1), True) for a in (Q, K, V))
  m = None if qm is None else _cu(qm)
  O, P = ops.attention_core(tq, tk, tv, H, query_mask=m, causal=causal, return_scores=True)
  O.backward(_cu(dO.reshape(B, T, -1)))
  with torch.no_grad():
    O0, P0 = ops.attention_core(tq, tk, tv, H, query_mask=m, causal=causal, return_scores=True)
  assert _bits_equal(P, P0) and _bits_equal(O, O0), "grad and no-grad calls differ"
  sh = lambda t, L, d: t.reshape(B, L, H, d)
  return (sh(O.detach(), T, V.shape[-1]), P, sh(tq.grad, T, Q.shape[-1]), sh(tk.grad, S, Q.shape[-1]),
          sh(tv.grad, S, V.shape[-1]))


def _core_case(B, T, S, H, dk, dv, causal=False, masked_rows=True, seed=0):
  Q, K, V, dO = _core_inputs(B, T, S, H, dk, dv, seed)
  qm = None
  if masked_rows:
    qm = np.ones((B, T), bool)
    qm[-1, ::3] = False                              # fully masked rows, real scores up to +-80
  got = _core_call(Q, K, V, dO, H, qm, causal)
  keep = ao.combined_mask(B, T, S, query_mask=qm, causal=causal)
  q, k, v, g = (a.astype(np.float64) for a in (Q, K, V, dO))
  eO, eP, Qs = ao.core_forward(q, k, v, keep)
  edQ, edK, edV = ao.core_backward(q, k, v, eP, Qs, g)
  bd = ao.core_error_bounds(q, k, v, eP, Qs, g)
  where = f"B={B} T={T} S={S} H={H} dk={dk} dv={dv} causal={causal}"
  for name, x, e in zip(("O", "P", "dQ", "dK", "dV"), got, (eO, eP, edQ, edK, edV)):
    _rows(f"{name} ({where})", x, e, bd[name])


@pytest.mark.parametrize("dk,dv", cases.width_pairs())
def test_core_at_every_width_and_tile_edge(dk, dv):
  for i, (T, S, k, v) in enumerate(c for c in cases.core_tile_cases() if c[2:] == (dk, dv)):
    _core_case(3, T, S, 2, dk, dv, causal=i % 2 == 1, seed=i)


@pytest.mark.parametrize("T,S", [(1, 3), (3, 1), (5, 1), (1, 2), (2, 1)])
def test_core_one_and_two_row_tiles_at_128(T, S):
  assert cases.plan(1, 256)[1] == 2 and cases.plan(1, 259)[1] == 1
  for H in (1, 16):
    _core_case(3, T, S, H, 128, 128, seed=H)


PACKED = [(B, H, T, d) for i, (B, H, T) in enumerate(cases.packing_cases())
          for d in [[(16, 16), (7, 9), (33, 65), (128, 128)][i % 4]]]


@pytest.mark.parametrize("B,H,T,d", PACKED)
def test_core_packed_ctas_and_dead_teams(B, H, T, d):
  for S in (1, 5, cases.plan(T, sum(d))[1] + 1):
    _core_case(B, T, S, H, *d, causal=S == 5, seed=B * H * T + S)


def _poisoned(arrays, H, n, names):
  """copies of the named arrays with sequence n = b H + h set to NaN"""
  b, h = divmod(n, H)
  out = dict(arrays)
  for k in names:
    out[k] = arrays[k].copy()
    out[k][b, :, h] = np.nan
  return out


def _same_elsewhere(name, clean, dirty, seq_axes, n, H):
  """Every sequence but n = b H + h (b, h on axes `seq_axes`) bitwise unchanged; n's own rows are poisoned."""
  b, h = divmod(n, H)
  c, d = clean.detach().cpu().numpy(), dirty.detach().cpu().numpy()
  idx = [slice(None)] * c.ndim
  idx[seq_axes[0]], idx[seq_axes[1]] = b, h
  others = np.ones(c.shape, bool)
  others[tuple(idx)] = False
  assert np.array_equal(c.view(np.uint32)[others], d.view(np.uint32)[others]), f"{name}: another sequence changed"
  assert np.isnan(d[tuple(idx)]).all(), f"{name}: the poison did not reach its own sequence"


ISOLATION = [(2, 16, 1, 9, 16, 16), (3, 11, 1, 4, 7, 9), (7, 5, 3, 70, 33, 17), (1, 16, 2, 3, 128, 128),
             (31, 1, 1, 17, 8, 8)]


@pytest.mark.parametrize("B,H,T,S,dk,dv", ISOLATION)
def test_core_sequences_in_one_cta_stay_apart(B, H, T, S, dk, dv):
  Q, K, V, dO = _core_inputs(B, T, S, H, dk, dv, seed=S)
  base = dict(Q=Q, K=K, V=V, dO=dO)
  clean = _core_call(Q, K, V, dO, H, None, True)
  axes = {"O": (0, 2), "P": (0, 1), "dQ": (0, 2), "dK": (0, 2), "dV": (0, 2)}
  for n in {0, (B * H) // 2, B * H - 1}:
    for names in (("K", "V"), ("Q", "dO")):
      a = _poisoned(base, H, n, names)
      dirty = _core_call(a["Q"], a["K"], a["V"], a["dO"], H, None, True)
      for name, c, d in zip(("O", "P", "dQ", "dK", "dV"), clean, dirty):
        _same_elsewhere(f"{name} (poisoned {names} of sequence {n})", c, d, axes[name], n, H)


# ---- C. the dense modes ----------------------------------------------------------------------------------------------
def _dense_data(B, Tq, Tv, dim, dv, mode, seed):
  rng = np.random.RandomState(seed)
  u = dim ** -0.25                                 # q . k of order 1, as in tests/test_gpu_dense_attention.py
  q = (rng.normal(size=(B, Tq, dim)) * u).astype(np.float32)
  k = (rng.normal(size=(B, Tv, dim)) * u).astype(np.float32)
  v = rng.normal(size=(B, Tv, dv)).astype(np.float32)
  g = rng.normal(size=(B, Tq, dv)).astype(np.float32)
  if mode == "additive":
    lim = np.sqrt(3.0 / dim)
    scale = rng.uniform(-lim, lim, size=(dim,)).astype(np.float32)
  else:
    scale = np.array(rng.uniform(0.5, 1.5), np.float32)
  cw = np.array(rng.uniform(0.5, 1.5), np.float32) if mode == "concat" else None
  return q, k, v, g, scale, cw


def _dense_call(mode, q, k, v, g, scale, cw, qm, vm, causal, rate, seed, call):
  tq, tk, tv, ts, tw = (_cu(a, True) for a in (q, k, v, scale, cw))
  mk = lambda m: None if m is None else _cu(m)
  out, w = ops.dense_attention(tq, tk, tv, mode, ts, tw, query_mask=mk(qm), value_mask=mk(vm), causal=causal,
                               rate=rate, seed=seed, call=call, return_scores=True)
  out.backward(_cu(g))
  with torch.no_grad():
    _, w0 = ops.dense_attention(tq, tk, tv, mode, ts, tw, query_mask=mk(qm), value_mask=mk(vm), causal=causal,
                                rate=rate, seed=seed, call=call, return_scores=True)
  assert _bits_equal(w, w0), "grad and no-grad weights differ"
  return out, w, tq.grad, tk.grad, tv.grad, ts.grad, (tw.grad if tw is not None else None)


def _dense_case(mode, B, Tq, Tv, dim, dv, qm=None, vm=None, causal=False, rate=0.0, seed=7, call=1, seed_data=0):
  q, k, v, g, scale, cw = _dense_data(B, Tq, Tv, dim, dv, mode, seed_data)
  out, w, dq, dk, dv_, dscale, dwc = _dense_call(mode, q, k, v, g, scale, cw, qm, vm, causal, rate, seed, call)
  keep = ro.dropout_keep((B, Tq, Tv), rate, seed, call) if rate else None
  eo, ew, cache = dao.forward(q, k, v, mode, scale, cw, qm, vm, causal, keep, rate)
  edq, edk, edv, edscale, edwc = dao.backward(cache, g)
  bd = dao.error_bounds(cache, g)
  where = f"{mode} B={B} Tq={Tq} Tv={Tv} dim={dim} dv={dv} causal={causal} rate={rate}"
  for name, x, e in zip(("out", "weights", "dq", "dk", "dv"), (out, w, dq, dk, dv_), (eo, ew, edq, edk, edv)):
    _rows(f"{name} ({where})", x, e, bd[name])
  if rate:
    wn = w.detach().cpu().numpy()
    assert np.all(wn[~keep] == 0) and not np.signbit(wn[~keep]).any(), f"a dropped weight is not +0 ({where})"
    assert np.all(wn[keep & (ew > 0)] > 0), f"a kept weight is 0 ({where})"
  mag_scale, mag_wc = dao.weight_grad_magnitudes(cache, g)
  err = np.abs(_np(dscale).reshape(np.shape(edscale)) - edscale)
  assert np.all(err <= 1e-5 * np.asarray(mag_scale)), f"dscale ({where}): error {np.max(err):.3g}"
  if mode == "concat":
    assert abs(float(dwc) - edwc) <= 1e-5 * mag_wc, f"dconcat_weight ({where}): error {abs(float(dwc) - edwc):.3g}"


@pytest.mark.parametrize("mode", dao.MODES)
@pytest.mark.parametrize("dim,dv", cases.DENSE_WIDTHS)
def test_dense_dropout_at_every_tile_edge(mode, dim, dv):
  for i, (B, Tq, Tv, d, e) in enumerate(c for c in cases.dense_dropout_cases() if c[3:] == (dim, dv)):
    rng = np.random.RandomState(i)
    qm = rng.rand(B, Tq) < 0.8 if i % 2 else None
    vm = rng.rand(B, Tv) < 0.8 if i % 3 else None
    _dense_case(mode, B, Tq, Tv, dim, dv, qm=qm, vm=vm, rate=0.3, call=i, seed_data=i)


@pytest.mark.parametrize("mode", dao.MODES)
def test_dense_causal_with_unequal_lengths(mode):
  for i, (B, Tq, Tv, dim, dv) in enumerate(cases.dense_causal_cases()):
    _dense_case(mode, B, Tq, Tv, dim, dv, causal=True, seed_data=i)
    vm = np.ones((B, Tv), bool)
    vm[0, 0] = False                               # causal row 0 of batch 0 keeps only key 0: fully masked
    vm[1] = False                                  # every row of batch 1 fully masked
    qm = np.ones((B, Tq), bool)
    qm[2, ::2] = False                             # output-masked rows
    _dense_case(mode, B, Tq, Tv, dim, dv, qm=qm, vm=vm, causal=True, rate=0.2 if i % 2 else 0.0, call=i,
                seed_data=i + 100)


@pytest.mark.parametrize("mode", dao.MODES)
def test_dense_sequences_in_one_cta_stay_apart(mode):
  B, Tq, Tv, dim, dv = 9, 3, 5, 32, 24
  q, k, v, g, scale, cw = _dense_data(B, Tq, Tv, dim, dv, mode, 3)
  args = (None, None, False, 0.3, 11, 2)
  clean = _dense_call(mode, q, k, v, g, scale, cw, *args)[:5]
  for b in (0, 4, 8):
    for names in (("k", "v"), ("q", "g")):
      a = dict(q=q, k=k, v=v, g=g)
      for n in names:
        a[n] = a[n].copy()
        a[n][b] = np.nan
      dirty = _dense_call(mode, a["q"], a["k"], a["v"], a["g"], scale, cw, *args)[:5]
      for name, c, d in zip(("out", "weights", "dq", "dk", "dv"), clean, dirty):
        c, d = c.detach().cpu().numpy(), d.detach().cpu().numpy()
        others = np.arange(B) != b
        assert np.array_equal(c[others].view(np.uint32), d[others].view(np.uint32)), \
            f"{mode} {name}: poisoned {names} of batch {b} changed another batch"
