"""Edge cases of the in-batch softmax loss on the tensor cores (csrc/softmax_tc.cu forward, csrc/softmax_tc_bwd.cu backward,
operand images from csrc/tc_split.cuh, option operands from csrc/softmax_ext.cuh) and of the exact CUDA-core path
(csrc/softmax.cu) it hands over to: routing and head-dim edges, the candidate-part schedule and the dX drain, confident and
flat logit rows, weights and grad_loss across the exponent range, every option mode, power-of-two scale equivariance, and
the exact kernels with more than one row block.

The reference is float64 of the same formula (torch float64, on the device the inputs live on, in row blocks):
  l_ij = s_ij / T + b_j,  s = q . c^T,  b the candidate bias (0 without one); only kept entries count (a masked entry or an
  accidental hit is left out of the sum; a masked positive has l_ii = MIN_FLOAT); p_ij = exp(l_ij - lse_i);
  G_ij = (p_ij - [i = j]) w_i g / T over kept entries, 0 elsewhere;  dq = G . c,  dc = G^T . q.
Bars (DESIGN section 2, "Softmax bars"):
  E_ij  bar (E) of the split product q . c^T: 1e-5 (|q| |c|^T)_ij + 2^-36 (amax_q sum_k |c_jk| + amax_c sum_k |q_ik|).
  e_ij  = E_ij / T + 2^-22 (|l_ij| + |b_j|): the logit error (the 2^-22 term covers the fp32 scale, the log2(e) conversion
        and the bias FMA).
  (L)   |lse_i - ref| <= max_{j kept} e_ij + eps_i.  logsumexp is 1-Lipschitz in the max-norm of the logits.
        eps_i = 2^-21 n + 2^-19 + 2^-22 (|lse_i| + 1) + C 2^-126, n = tiles per part + 2 parts (tensor cores) or
        ceil(C / 256) + 13 adds (exact path).  A term of the sum carries the ex2.approx.ftz error (2^-22 relative, PTX ISA)
        and 16 sequential fp32 adds in its tile half (8 per column parity, then the two sums and the running sum); every
        later tile of the part rescales the running sum (one ex2, one multiply, one add: <= 2^-21); the quad merge is two
        such steps, the combine one exp2f, one multiply and one add per (part, half) partial: 2^-19 covers the fixed part.
        The final (M + log2 L) ln2 is three roundings of lse (2^-22 |lse|); ex2 results below 2^-126 flush to 0 (C 2^-126).
  loss  |loss - ref| <= sum_i |w_i| (L_i + e_ii) + 2^-21 |w_i row_i| + 2^-24 |loss|  (five fp32 roundings of each row
        term; the fp64 reduction adds nothing worth counting; e_ii = 2^-22 |MIN_FLOAT| for a masked positive).
  (G)   per element of dq and dc, with a_i = |w_i g / T| and the backward's exponent argument rounded once more
        (e'_ij = e_ij + 2^-22 (|lse_i| + 10)):
          dP_ij  = p_ij (expm1(e'_ij + L_i) + 2^-21)            (lse off by L_i, logit by e'_ij, ex2 and the hi/lo split of G)
          bar_dq = a (.) (dP . |c|) + 2^-39 a (.) sum_j |c_j| + E(G, c)
          bar_dc = dP^T . (a (.) |q|) + 2^-38 max_i a_i sum_i |q_i| + E(G^T, q)
        The 2^-39 / 2^-38 terms are the hi/lo split's absolute floor (half the fp16 subnormal spacing at the 2^14 scale G
        carries: in units of p for the dq launch, of max |w| for the dc launch); E restarts every 192 accumulation steps.
        The bar is relative to p, so it is tight on confident rows (G_ii = p_ii - 1 cancels), small weights and masked
        entries, where a per-tensor bar is not.  The exact path's products are fp32 FMA chains as long as the reduction:
        there the 1e-5 of E(G, .) becomes 1.01 * 2^-24 * (C for dq, B for dc) when that is larger.
  (B)   bitwise, where every value involved is a normal fp32 number: (q 2^k, c 2^-k) gives the loss and lse bits, dq 2^-k
        and dc 2^k; (q 2^k, 1/T 2^-k) gives the loss bits; w 2^k scales the loss and both gradients by 2^k, grad_loss 2^k
        both gradients; two calls and a workspace full of NaN-payload sentinels give the same bits.
The GPU tests are marked one by one; the bar self-tests at the top run without a GPU.
"""
import ctypes
import math

import numpy as np
import pytest
import torch

gpu = pytest.mark.gpu

SENTINEL = 0x7FC01234        # a NaN with a payload: a buffer the kernels overwrite cannot keep these bits by accident
MIN_FLOAT = float(np.float32(np.finfo(np.float32).min / 100.0))
FLT_MIN = float(np.finfo(np.float32).tiny)
FLT_MAX = float(np.finfo(np.float32).max)
F64 = torch.float64


# ------------------------------------------------------------------------------------------------
# The schedule, restated: how many candidate parts each launch cuts its streamed tiles into
# ------------------------------------------------------------------------------------------------
def _cdiv(a, b):
  return -(-a // b)


def stream_parts(n_blocks, n_tiles, sms):
  """tc_split.cuh stream_parts: minimise waves x (tiles per CTA + 6)."""
  parts, best = 1, 1e30
  for c in range(1, min(16, n_tiles) + 1):
    cost = _cdiv(n_blocks * c, sms) * (_cdiv(n_tiles, c) + 6.0)
    if cost < best * 0.97:
      best, parts = cost, c
  return parts


def part_tiles(n_tiles, parts):
  """Tile counts of the parts: part k streams tiles [k n / parts, (k + 1) n / parts)."""
  return sorted({(k + 1) * n_tiles // parts - k * n_tiles // parts for k in range(parts)})


def schedule(B, C, sms):
  nct, qt = _cdiv(C, 128), _cdiv(B, 128)
  pf, pq, pc = stream_parts(_cdiv(B, 256), nct, sms), stream_parts(qt, nct, sms), stream_parts(nct, qt, sms)
  return {"fwd": (pf, part_tiles(nct, pf)), "dq": (pq, part_tiles(nct, pq)), "dc": (pc, part_tiles(qt, pc))}


def chain_tc(B, C, sms):
  parts, tiles = schedule(B, C, sms)["fwd"]
  return max(tiles) + 2 * parts


def chain_exact(C):
  return _cdiv(C, 256) + 13


def rel_exact(n):
  return max(1e-5, 1.01 * n * 2.0 ** -24)


# ------------------------------------------------------------------------------------------------
# float64 reference and bars
# ------------------------------------------------------------------------------------------------
class Ref:
  pass


def reference(q, c, inv_t, w=None, bias=None, ids=None, mask=None, g=1.0, chain=1, rel=(1e-5, 1e-5), grads=True,
              keep_g=False):
  """lse, loss, dq, dc in float64 with the bars of the module docstring, in row blocks of <= 2^26 entries."""
  dev = q.device
  q64, c64 = q.detach().to(F64), c.detach().to(F64)
  B, d = q64.shape
  C = c64.shape[0]
  w64 = torch.ones(B, dtype=F64, device=dev) if w is None else w.detach().to(F64).reshape(-1)
  b64 = torch.zeros(C, dtype=F64, device=dev) if bias is None else bias.detach().to(F64).reshape(-1)
  aq, ac = q64.abs(), c64.abs()
  amax_q, amax_c = aq.max(), ac.max()
  rs_q, rs_c, cs_q, cs_c = aq.sum(1), ac.sum(1), aq.sum(0), ac.sum(0)
  fac = w64 * (float(g) * inv_t)
  a = fac.abs()
  r = Ref()
  r.lse = torch.empty(B, dtype=F64, device=dev); r.barL = torch.empty_like(r.lse)
  row = torch.empty_like(r.lse); e_pos = torch.empty_like(r.lse)
  if grads:
    r.dq = torch.zeros((B, d), dtype=F64, device=dev); r.bar_dq = torch.zeros_like(r.dq)
    r.dc = torch.zeros((C, d), dtype=F64, device=dev); r.bar_dc = torch.zeros_like(r.dc)
    gsum_r = torch.zeros(B, dtype=F64, device=dev); gsum_c = torch.zeros(C, dtype=F64, device=dev)
    amax_g = torch.zeros((), dtype=F64, device=dev)
  if keep_g:
    r.G, r.l, r.keep = [], [], []
  cols = torch.arange(C, device=dev)
  blk = max(1, min(B, (1 << 26) // C))
  for r0 in range(0, B, blk):
    r1 = min(B, r0 + blk)
    rows = torch.arange(r0, r1, device=dev)
    E = 1e-5 * (aq[r0:r1] @ ac.T) + 2.0 ** -36 * (amax_q * rs_c[None, :] + amax_c * rs_q[r0:r1, None])
    l = (q64[r0:r1] @ c64.T) * inv_t + b64[None, :]
    diag = cols[None, :] == rows[:, None]
    keep = torch.ones_like(diag) if mask is None else mask[r0:r1].to(dev).bool()
    if ids is not None:
      idv = ids.to(dev)
      keep = keep & ~((idv[None, :] == idv[r0:r1, None]) & ~diag)
    e = abs(inv_t) * E + 2.0 ** -22 * (l.abs() + b64.abs()[None, :])
    lk = torch.where(keep, l, torch.full_like(l, -math.inf))
    m = lk.max(1).values
    has = torch.isfinite(m)
    ms = torch.where(has, m, torch.zeros_like(m))
    lse = torch.where(has, ms + torch.log(torch.exp(lk - ms[:, None]).sum(1)), torch.full_like(m, MIN_FLOAT + math.log(C)))
    kii = keep.gather(1, rows[:, None]).squeeze(1)
    pos = torch.where(kii, l.gather(1, rows[:, None]).squeeze(1), torch.full_like(m, MIN_FLOAT))
    e_pos[r0:r1] = torch.where(kii, e.gather(1, rows[:, None]).squeeze(1), torch.full_like(m, 2.0 ** -22 * abs(MIN_FLOAT)))
    eps = 2.0 ** -21 * chain + 2.0 ** -19 + 2.0 ** -22 * (lse.abs() + 1) + C * 2.0 ** -126
    barL = torch.where(keep, e, torch.zeros_like(e)).max(1).values + eps
    r.lse[r0:r1], r.barL[r0:r1], row[r0:r1] = lse, barL, lse - pos
    if not grads:
      continue
    p = torch.where(keep, torch.exp(l - lse[:, None]), torch.zeros_like(l))
    G = (p - (diag & keep).to(F64)) * fac[r0:r1, None]
    ep = e + 2.0 ** -22 * (lse.abs()[:, None] + 10)
    dP = torch.where(keep, p * (torch.expm1(ep + barL[:, None]).clamp(max=1e300) + 2.0 ** -21), torch.zeros_like(p))
    Ga = G.abs()
    r.dq[r0:r1] = G @ c64
    r.bar_dq[r0:r1] = a[r0:r1, None] * (dP @ ac + 2.0 ** -39 * cs_c[None, :]) + rel[0] * (Ga @ ac)
    r.dc += G.T @ q64[r0:r1]
    r.bar_dc += dP.T @ (a[r0:r1, None] * aq[r0:r1]) + rel[1] * (Ga.T @ aq[r0:r1])
    gsum_r[r0:r1] = Ga.sum(1); gsum_c += Ga.sum(0); amax_g = torch.maximum(amax_g, Ga.max())
    if keep_g:
      r.G.append(G); r.l.append(l); r.keep.append(keep)
  wr = w64 * row
  r.loss = float(wr.sum())
  r.bar_loss = float((w64.abs() * (r.barL + e_pos) + 2.0 ** -21 * wr.abs()).sum()) + 2.0 ** -24 * abs(r.loss)
  if grads:
    r.bar_dq += 2.0 ** -36 * (amax_g * cs_c[None, :] + amax_c * gsum_r[:, None]) + 16 * 2.0 ** -149
    r.bar_dc += (2.0 ** -36 * (amax_g * cs_q[None, :] + amax_q * gsum_c[:, None]) + 2.0 ** -38 * a.max() * cs_q[None, :] +
                 16 * 2.0 ** -149)
  if keep_g:
    r.G, r.l, r.keep = torch.cat(r.G), torch.cat(r.l), torch.cat(r.keep)
  return r


def check(got, ref, bar, what):
  """Per-element bar: returns the worst err / bar; on a miss, names the first element that misses."""
  ref = torch.as_tensor(ref, dtype=F64)
  got = torch.as_tensor(got).detach().to(device=ref.device, dtype=F64)
  bar = torch.as_tensor(bar, dtype=F64, device=ref.device)
  assert torch.isfinite(ref).all(), f"{what}: the reference is not finite"
  assert not torch.isnan(bar).any(), f"{what}: the bar is NaN"
  fin = torch.isfinite(got)
  assert fin.all(), f"{what}: {int((~fin).sum())} non-finite results"
  err = (got - ref).abs()
  ratio = torch.where(bar > 0, err / bar, torch.where(err > 0, torch.full_like(err, math.inf), torch.zeros_like(err)))
  worst = float(ratio.max())
  bad = err > bar
  if bool(bad.any()):
    i = tuple(int(v) for v in torch.nonzero(bad)[0]) if bad.dim() else ()
    raise AssertionError(f"{what}: {int(bad.sum())} of {bad.numel()} elements miss the bar, worst err/bar {worst:.3g}; first "
                         f"{i}: got {float(got[i])!r} ref {float(ref[i])!r} err {float(err[i]):.3e} bar {float(bar[i]):.3e}")
  print(f"softmax-bars {what}: worst err/bar {worst:.3g}")
  return worst


def check_all(r, what, loss=None, lse=None, dq=None, dc=None):
  out = {}
  if lse is not None:
    out["lse"] = check(lse, r.lse, r.barL, f"{what} (L)")
  if loss is not None:
    out["loss"] = check(torch.as_tensor(float(loss), dtype=F64), torch.tensor(r.loss, dtype=F64),
                        torch.tensor(r.bar_loss, dtype=F64), f"{what} loss")
  if dq is not None:
    out["dq"] = check(dq, r.dq, r.bar_dq, f"{what} dq (G)")
  if dc is not None:
    out["dc"] = check(dc, r.dc, r.bar_dc, f"{what} dc (G)")
  return out


# ------------------------------------------------------------------------------------------------
# The bars have teeth (no GPU): they accept the float64 answer rounded to fp32 and reject planted defects
# ------------------------------------------------------------------------------------------------
def _cpu_case(seed, B=300, C=400, d=16, masked=False):
  g = torch.Generator().manual_seed(seed)
  q = torch.nn.functional.normalize(torch.randn((B, d), generator=g), dim=1)
  c = torch.nn.functional.normalize(torch.cat([q, torch.randn((C - B, d), generator=g)]) +
                                    0.5 * torch.randn((C, d), generator=g), dim=1)
  w = torch.rand(B, generator=g) + 0.5
  mask = (torch.rand((B, C), generator=g) > 0.2) if masked else None
  return q, c, w, mask


def test_bars_accept_the_rounded_float64_answer():
  q, c, w, mask = _cpu_case(1, masked=True)
  r = reference(q, c, 20.0, w, mask=mask, chain=4)
  check_all(r, "rounded float64", loss=np.float32(r.loss), lse=r.lse.float(), dq=r.dq.float(), dc=r.dc.float())


def test_bars_reject_a_missing_column_tile():
  q, c, w, _ = _cpu_case(2)
  r = reference(q, c, 20.0, w, chain=4, keep_g=True)
  G = r.G.clone(); G[:, 128:256] = 0
  with pytest.raises(AssertionError, match="dq"):
    check(G @ c.to(F64), r.dq, r.bar_dq, "dq without tile 1")


def test_bars_reject_an_lse_off_by_four_bars():
  q, c, w, _ = _cpu_case(3)
  r = reference(q, c, 20.0, w, chain=4, grads=False)
  lse = r.lse.clone(); lse[37] += 4 * r.barL[37]
  with pytest.raises(AssertionError, match="lse"):
    check(lse.float(), r.lse, r.barL, "lse")


def test_bars_reject_an_unmasked_entry():
  q, c, w, mask = _cpu_case(4, masked=True)
  r = reference(q, c, 20.0, w, mask=mask, chain=4, keep_g=True)
  # the masked entry with the largest probability, given back its probability
  pm = torch.where(r.keep, torch.full_like(r.l, -math.inf), r.l - r.lse[:, None])
  i, j = (int(v) for v in divmod(int(pm.argmax()), pm.shape[1]))
  G = r.G.clone(); G[i, j] = math.exp(float(pm[i, j])) * float(w[i]) * 20.0
  with pytest.raises(AssertionError, match="dq"):
    check((G @ c.to(F64)).float(), r.dq, r.bar_dq, "dq with an unmasked entry")


def test_bars_reject_a_part_counted_twice():
  q, c, w, _ = _cpu_case(5)
  r = reference(q, c, 20.0, w, chain=4, keep_g=True)
  dc = r.dc + r.G[128:256].T @ q[128:256].to(F64)
  with pytest.raises(AssertionError, match="dc"):
    check(dc.float(), r.dc, r.bar_dc, "dc with query tile 1 twice")


def test_schedule_restatement():
  """stream_parts as the kernels size their launches (132 SMs, the H100 SXM): the regimes the GPU cases are named for."""
  s = schedule(512, 65536, 132)
  assert s["fwd"] == (16, [32]) and s["dc"] == (1, [4])
  assert schedule(128, 128, 132)["fwd"] == (1, [1])
  assert schedule(16384, 16384, 132) == {"fwd": (2, [64]), "dq": (1, [128]), "dc": (1, [128])}


def test_retrieval_routes_options_with_a_negative_temperature_to_the_score_matrix(monkeypatch):
  """Options are fused only for a positive temperature; otherwise the reference's op sequence runs (host logic only)."""
  from recommenders_b200 import ops, tasks
  calls = []
  monkeypatch.setattr(ops, "inbatch_softmax_loss", lambda *a, **k: (calls.append("fused"), torch.zeros(()))[1])
  monkeypatch.setattr(ops, "inbatch_softmax_bias_supported", lambda B, C, d: True)
  monkeypatch.setattr(ops, "scores", lambda q, c: (calls.append("scores"), q @ c.T)[1])
  q, c = torch.randn(8, 4), torch.randn(12, 4)
  prob = torch.full((12,), 0.1)
  tasks.Retrieval(temperature=-0.5)(q, c, candidate_sampling_probability=prob, compute_metrics=False)
  assert calls == ["scores"]
  calls.clear()
  tasks.Retrieval(temperature=0.5)(q, c, candidate_sampling_probability=prob, compute_metrics=False)
  assert calls == ["fused"]


# ------------------------------------------------------------------------------------------------
# GPU helpers
# ------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def ops():
  from recommenders_b200 import ops as o
  return o


@pytest.fixture(scope="module")
def sms():
  return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


def _gen(seed):
  g = torch.Generator(device="cuda"); g.manual_seed(seed)
  return g


def _randn(shape, seed, scale=1.0):
  return torch.randn(shape, generator=_gen(seed), device="cuda") * scale


def _unit(x):
  return torch.nn.functional.normalize(x, dim=1)


def _pairs(B, C, d, seed, noise=0.5):
  """Unit-norm queries and candidates, candidate i near query i (the positive), the rest random."""
  q = _unit(_randn((B, d), seed))
  c = _unit(torch.cat([q, _randn((C - B, d), seed + 1)]) + noise / math.sqrt(d) * _randn((C, d), seed + 2))
  return q.contiguous(), c.contiguous()


def _away_from_zero(shape, seed):
  """Unit normal data with every |v| >= 2^-10: each 2^k-scaled copy with k in [-116, 124] is exact and normal."""
  v = _randn(shape, seed)
  return torch.where(v.abs() < 2.0 ** -10, torch.copysign(torch.full_like(v, 2.0 ** -10), v), v)


def _gl(g):
  return None if g is None else torch.tensor([g], dtype=torch.float32, device="cuda")


def _tc(ops, q, c, inv_t, w=None, bias=None, ids=None, mask=None, g=None, bwd=True):
  loss, lse = ops.inbatch_softmax_tc(q, c, w, inv_t, bias, ids, mask)
  if not bwd:
    return loss, lse, None, None
  dq, dc = ops.inbatch_softmax_tc_bwd(q, c, lse, w, inv_t, _gl(g), bias, ids, mask)
  return loss, lse, dq, dc


def _exact_fwd(ops, q, c, inv_t, w=None):
  B, d = q.shape; C = c.shape[0]
  loss = torch.empty((1,), device="cuda"); lse = torch.empty((B,), device="cuda")
  ws = torch.empty(ops.lib().tfrs_inbatch_softmax_workspace_bytes(B, C, d), dtype=torch.uint8, device="cuda")
  ops.check(ops.lib().tfrs_inbatch_softmax_fwd(ops.ptr(q), ops.ptr(c), B, C, d, ops.c_f(inv_t), ops.ptr(w), ops.ptr(loss),
                                               ops.ptr(lse), ops.ptr(ws), ws.numel(), ops.stream()), "inbatch_softmax_fwd")
  return loss.view(()), lse


def _verify(ops, sms, what, q, c, inv_t, w=None, bias=None, ids=None, mask=None, g=None, bwd=True):
  """Tensor-core forward (+ backward fed its lse) against the reference under (L), loss and (G)."""
  B, C = q.shape[0], c.shape[0]
  loss, lse, dq, dc = _tc(ops, q, c, inv_t, w, bias, ids, mask, g, bwd)
  r = reference(q, c, inv_t, w, bias, ids, mask, 1.0 if g is None else g, chain_tc(B, C, sms), grads=bwd)
  check_all(r, what, loss, lse, dq, dc)
  return r, (loss, lse, dq, dc)


class _Spy:
  """Counts the calls of the tensor-core entry points and keeps the forward's lse."""

  def __init__(self, ops, monkeypatch):
    self.fwd = self.bwd = 0
    self.lse = None
    f0, b0 = ops.inbatch_softmax_tc, ops.inbatch_softmax_tc_bwd

    def fwd(*a, **k):
      self.fwd += 1
      out = f0(*a, **k)
      self.lse = out[1]
      return out

    def bwd(*a, **k):
      self.bwd += 1
      return b0(*a, **k)
    monkeypatch.setattr(ops, "inbatch_softmax_tc", fwd)
    monkeypatch.setattr(ops, "inbatch_softmax_tc_bwd", bwd)


def _autograd(ops, q, c, w, T, **kw):
  qg, cg = q.clone().requires_grad_(True), c.clone().requires_grad_(True)
  loss = ops.inbatch_softmax_loss(qg, cg, w, T, **kw)
  loss.backward()
  return loss.detach(), qg.grad, cg.grad


# ------------------------------------------------------------------------------------------------
# 1. Route and kernel edges
# ------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("B", [511, 512])
def test_route_at_512(ops, sms, monkeypatch, B):
  """The same data on both sides of SOFTMAX_TC_MIN_B: exact path at 511, tensor cores at 512."""
  q, c = _pairs(512, 640, 48, 101)
  q, c = q[:B].contiguous(), c[:B + 128].contiguous()
  w = torch.rand(B, generator=_gen(102), device="cuda") + 0.5
  spy = _Spy(ops, monkeypatch)
  loss, dq, dc = _autograd(ops, q, c, w, 0.05)
  tc = B >= 512
  assert (spy.fwd, spy.bwd) == ((1, 1) if tc else (0, 0))
  C = c.shape[0]
  r = reference(q, c, 20.0, w, chain=chain_tc(B, C, sms) if tc else chain_exact(C),
                rel=(1e-5, 1e-5) if tc else (rel_exact(C), rel_exact(B)))
  check_all(r, f"route B={B}", loss, spy.lse, dq, dc)


@gpu
@pytest.mark.parametrize("d", [1, 8, 63, 64, 65, 96, 127, 128, 129])
def test_route_head_dims(ops, sms, monkeypatch, d):
  """Forward on the tensor cores up to d = 128 (K slabs of 64: KB = 1, 2), backward up to 64; beyond that the exact
  kernels.  d in 65..128 runs the exact backward on the tensor-core lse (d = 96 among them)."""
  B, C = 512, 700
  q, c = _pairs(B, C, d, 111 + d)
  w = torch.rand(B, generator=_gen(112), device="cuda") + 0.5
  spy = _Spy(ops, monkeypatch)
  loss, dq, dc = _autograd(ops, q, c, w, 0.1)
  assert spy.fwd == (1 if d <= 128 else 0) and spy.bwd == (1 if d <= 64 else 0)
  r = reference(q, c, 10.0, w, chain=chain_tc(B, C, sms) if d <= 128 else chain_exact(C),
                rel=(1e-5, 1e-5) if d <= 64 else (rel_exact(C), rel_exact(B)))
  check_all(r, f"route d={d}", loss, spy.lse, dq, dc)


@gpu
@pytest.mark.parametrize("B,C", [(513, 513), (639, 639), (767, 767), (600, 601), (600, 727), (600, 728), (600, 729)])
def test_shape_edges(ops, sms, B, C):
  """Partial last query block and candidate tile; C - B of 1, 127, 128, 129."""
  q, c = _pairs(B, C, 40, 121)
  w = torch.rand(B, generator=_gen(122), device="cuda") + 0.5
  _verify(ops, sms, f"shape B={B} C={C}", q, c, 20.0, w)


# ------------------------------------------------------------------------------------------------
# 2. Schedule edges
# ------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("B,C,parts", [(128, 128, 1), (1024, 16896, None), (512, 65536, 16)])
def test_forward_parts(ops, sms, B, C, parts):
  """One part (a single candidate tile), a middle count, and the maximum of 16 parts."""
  pf, _ = schedule(B, C, sms)["fwd"]
  if parts is None:
    assert 2 < pf < 16, pf
  else:
    assert pf == parts, pf
  q, c = _pairs(B, C, 64, 131)
  w = torch.rand(B, generator=_gen(132), device="cuda") + 0.5
  _verify(ops, sms, f"fwd parts={pf} B={B} C={C}", q, c, 20.0, w)


@gpu
def test_dq_parts_with_one_dc_part(ops, sms):
  """dq streams 128 candidate tiles in several parts and reduce_parts folds them; dc streams 4 query tiles in one part."""
  B, C = 512, 16384
  s = schedule(B, C, sms)
  assert s["dq"][0] > 1 and s["dc"][0] == 1, s
  q, c = _pairs(B, C, 64, 141)
  w = torch.rand(B, generator=_gen(142), device="cuda") + 0.5
  _verify(ops, sms, f"dq parts={s['dq'][0]}", q, c, 20.0, w)


@gpu
@pytest.mark.parametrize("B,tiles", [(1024, 8), (1025, 9), (1920, 15)])
def test_drain_edges(ops, sms, B, tiles):
  """The dX chain restarts every SB_DRAIN = 8 tiles: a dc part of 8k tiles drains on its last tile, 8k + 1 drains a
  one-tile chain, 8k + 7 a seven-tile chain.  The dq parts of these shapes hold 8 / 9 and 16 / 17 tiles."""
  C = 16896
  s = schedule(B, C, sms)
  assert s["dc"] == (1, [tiles]), s
  q, c = _pairs(B, C, 64, 151)
  w = torch.rand(B, generator=_gen(152), device="cuda") + 0.5
  _verify(ops, sms, f"drain dc tiles={tiles} dq tiles={s['dq'][1]}", q, c, 20.0, w)


@gpu
def test_cfg3(ops, sms):
  """B = C = 16384, d = 64 (bench cfg3): unit-norm rows at T = 0.05, weights in [0.5, 1.5)."""
  B = C = 16384
  q, c = _pairs(B, C, 64, 161)
  w = torch.rand(B, generator=_gen(162), device="cuda") + 0.5
  _verify(ops, sms, "cfg3", q, c, 20.0, w)


# ------------------------------------------------------------------------------------------------
# 3. Logit regimes
# ------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("T", [0.1, 0.05, 0.02])
def test_unit_norm_temperatures(ops, sms, T):
  """Unit-norm embeddings at the usual retrieval temperatures: many confident rows, where G_ii = p_ii - 1 cancels."""
  B, C = 1024, 1536
  q, c = _pairs(B, C, 64, 171, noise=0.3)
  r, _ = _verify(ops, sms, f"unit-norm T={T}", q, c, 1.0 / T, None)
  if T <= 0.05:
    confident = float(((r.lse - (q.double() * c[:B].double()).sum(1) / T) < 1e-3).float().mean())
    assert confident > 0.1, f"only {confident:.3f} of the rows have p_ii > 0.999"


@gpu
@pytest.mark.parametrize("case", ["near_uniform", "positive_far_below", "duplicate_candidates"])
def test_logit_shapes(ops, sms, case):
  B, C, d = 768, 1000, 64
  q, c = _pairs(B, C, d, 181)
  inv_t = 20.0
  if case == "near_uniform":
    q = q * 1e-4
  elif case == "positive_far_below":
    c = c.clone(); c[:B:3] = -q[::3]                     # every third positive is the least similar candidate
  else:
    c = c.clone(); c[1::2] = c[0::2][:c[1::2].shape[0]]  # exact ties: every odd candidate repeats the even one before
  w = torch.rand(B, generator=_gen(182), device="cuda") + 0.5
  _verify(ops, sms, case, q.contiguous(), c.contiguous(), inv_t, w)


@gpu
@pytest.mark.parametrize("case", ["zero_and_negative", "span_2^-40", "one_large"])
def test_weights(ops, sms, case):
  B, C = 1024, 1024
  q, c = _pairs(B, C, 64, 191)
  g = _gen(192)
  if case == "zero_and_negative":
    w = torch.rand(B, generator=g, device="cuda") * 2 - 1; w[::7] = 0
  elif case == "span_2^-40":
    w = torch.exp2(-40 * torch.rand(B, generator=g, device="cuda")); w[0] = 1.0
  else:
    w = torch.ones(B, device="cuda"); w[517] = 1e4
  _verify(ops, sms, f"weights {case}", q, c, 20.0, w)


@gpu
@pytest.mark.parametrize("g", [-1.0, 2.0 ** 40, 2.0 ** -40])
def test_grad_loss(ops, sms, g):
  B, C = 1024, 1100
  q, c = _pairs(B, C, 64, 201)
  w = torch.rand(B, generator=_gen(202), device="cuda") + 0.5
  _verify(ops, sms, f"grad_loss {g:g}", q, c, 20.0, w, g=g)


# ------------------------------------------------------------------------------------------------
# 4. Option modes (bias, ids, mask, all three): forward at KB = 1 and 2, backward at KB = 1
# ------------------------------------------------------------------------------------------------
I64_MIN, I64_MAX = -(1 << 63), (1 << 63) - 1


def _ids(B, C, seed):
  ids = np.random.RandomState(seed).permutation(10 * C)[:C].astype(np.int64) + 1000
  ids[12], ids[400] = (1 << 32) + 5, (2 << 32) + 5         # equal low words, different high words: not a hit
  ids[14], ids[501] = -1, 0xFFFFFFFF                       # likewise, with a negative id
  ids[13], ids[500] = -5, -5                               # negative ids: a hit
  ids[10], ids[300] = I64_MIN, I64_MIN
  ids[11], ids[C - 2] = I64_MAX, I64_MAX
  ids[127] = ids[5]; ids[128] = ids[6]; ids[C - 1] = ids[7]   # duplicates of a positive at the tile edge and at C - 1
  return torch.from_numpy(ids).cuda()


def _mask(B, C, seed, masked_positive=True):
  m = torch.rand((B, C), generator=_gen(seed), device="cuda") > 0.15
  m[:, 200] = False                                        # a column masked for every row
  m[3, :] = False                                          # a fully masked row (its weight is 0)
  if masked_positive:
    m[9, 9] = False; m[B - 1, B - 1] = False               # masked positives
  return m.to(torch.uint8).contiguous()


def _bias(C, seed):
  p = torch.exp2(-30 * torch.rand(C, generator=_gen(seed), device="cuda"))
  p[::11] = 1.0                                            # exactly 1: no correction
  p[5::13] = 1e-9                                          # below the 1e-6 clip
  return -torch.log(torch.clamp(p, 1e-6, 1.0))


@gpu
@pytest.mark.parametrize("d", [48, 100])
@pytest.mark.parametrize("mode", ["bias", "ids", "mask", "all"])
def test_option_modes(ops, sms, mode, d):
  """B % 32 != 0 and C % 32 != 0 (the transposed mask pack's partial words).  d = 100 is the 128-wide K of the forward
  (softmax_tc_kernel<2, 1> / <2, 2>), reached through ops.inbatch_softmax_tc only."""
  B, C = 600, 777
  q, c = _pairs(B, C, d, 211)
  w = torch.rand(B, generator=_gen(212), device="cuda") + 0.5
  bias = _bias(C, 213) if mode in ("bias", "all") else None
  ids = _ids(B, C, 214) if mode in ("ids", "all") else None
  mask = None
  if mode in ("mask", "all"):
    mask = _mask(B, C, 215, masked_positive=mode == "mask")
    w[3] = 0.0
  r, _ = _verify(ops, sms, f"options {mode} d={d}", q, c, 10.0, w, bias, ids, mask, bwd=d <= 64)
  if mode == "mask":
    assert r.loss > 1e36, "the masked positives do not carry MIN_FLOAT"


# ------------------------------------------------------------------------------------------------
# 5. The fp32 exponent range
# ------------------------------------------------------------------------------------------------
def _bits(t):
  return t.detach().contiguous().view(torch.int32).cpu()


def _assert_scaled_bits(got, base, e, what, min_normal=0.25):
  """got == ldexp(base, e) bit for bit wherever that is a normal fp32 number."""
  want = torch.ldexp(base.double(), torch.tensor(float(e), dtype=F64, device=base.device))
  m = (want.abs() >= FLT_MIN) & (want.abs() <= FLT_MAX)
  assert float(m.double().mean()) >= min_normal, f"{what}: too few normal results to compare"
  diff = _bits(got)[m.cpu()] != _bits(want.float())[m.cpu()]
  assert not bool(diff.any()), f"{what}: {int(diff.sum())} of {int(m.sum())} normal results differ from the base call x 2^{e}"


EXP_PAIRS = [(0, -116), (-116, 0), (-60, 60), (60, -60), (-100, 0), (0, -100), (-50, -50), (50, -110), (-110, 50),
             (60, -100), (-100, 60), (8, 0), (0, 8)]


@gpu
@pytest.mark.parametrize("a,b", EXP_PAIRS)
def test_exponent_range(ops, sms, a, b):
  """q 2^a, c 2^b: (L) and (G) wherever the logits and the gradients have normal fp32 scales.  At max|c| near 2^-114 the
  dq factor w_i g / T 2^-(wexp + 14 + cexp) is about 2^-141, at max|q| near 2^-114 the dc factor about 2^-140: not normal
  numbers.  1/T and w are not powers of two, so such a factor would keep only its leading bits."""
  B, C, d = 1024, 1024, 64
  q, c = _away_from_zero((B, d), 221) * 2.0 ** a, _away_from_zero((C, d), 222) * 2.0 ** b
  w = torch.rand(B, generator=_gen(223), device="cuda") + 0.5
  inv_t = 1.3
  loss, lse, dq, dc = _tc(ops, q, c, inv_t, w)
  r = reference(q, c, inv_t, w, chain=chain_tc(B, C, sms))
  for name, t in [("logits", (q[:64].double() @ c.double().T) * inv_t), ("dq", r.dq), ("dc", r.dc)]:
    amax = float(t.abs().max())
    assert 2.0 ** -120 <= amax <= 2.0 ** 100, f"a={a} b={b}: {name} scale {amax:.3e} is outside the normal range"
  check_all(r, f"exponent a={a} b={b}", loss, lse, dq, dc)


@gpu
def test_scale_equivariance_bits(ops, sms):
  """(B): exact power-of-two relations between calls, including where the output factor is not a normal number.  At
  cfg3 size each backward launch streams all its tiles in one part: with several parts, a part's share of a result near
  2^-126 can be a subnormal number, and rounding it is not equivariant."""
  B, C, d = 16384, 16384, 64
  s = schedule(B, C, sms)
  assert s["dq"][0] == 1 and s["dc"][0] == 1, s
  q, c = _away_from_zero((B, d), 231), _away_from_zero((C, d), 232)
  w = torch.rand(B, generator=_gen(233), device="cuda") + 0.5
  inv_t = 4.0
  loss0, lse0, dq0, dc0 = _tc(ops, q, c, inv_t, w)
  for k in [-116, -100, -60, 40, 100, 116]:
    loss, lse, dq, dc = _tc(ops, q * 2.0 ** k, c * 2.0 ** -k, inv_t, w)
    assert torch.equal(_bits(loss), _bits(loss0)) and torch.equal(_bits(lse), _bits(lse0)), f"(q 2^{k}, c 2^{-k}) loss / lse"
    _assert_scaled_bits(dq, dq0, -k, f"(q 2^{k}, c 2^{-k}) dq")
    _assert_scaled_bits(dc, dc0, k, f"(q 2^{k}, c 2^{-k}) dc")
  for k in [-100, -40, 20]:
    loss, lse, dq, dc = _tc(ops, q * 2.0 ** k, c, inv_t * 2.0 ** -k, w)
    assert torch.equal(_bits(loss), _bits(loss0)), f"(q 2^{k}, 1/T 2^{-k}) loss"
    assert torch.equal(_bits(lse), _bits(lse0)), f"(q 2^{k}, 1/T 2^{-k}) lse"
    _assert_scaled_bits(dq, dq0, -k, f"(q 2^{k}, 1/T 2^{-k}) dq")
    assert torch.equal(_bits(dc), _bits(dc0)), f"(q 2^{k}, 1/T 2^{-k}) dc"
  for k in [-100, -60, 30, 60]:
    loss, lse, dq, dc = _tc(ops, q, c, inv_t, w * 2.0 ** k)
    _assert_scaled_bits(loss, loss0, k, f"w 2^{k} loss", 1.0)
    assert torch.equal(_bits(lse), _bits(lse0)), f"w 2^{k} lse"
    _assert_scaled_bits(dq, dq0, k, f"w 2^{k} dq")
    _assert_scaled_bits(dc, dc0, k, f"w 2^{k} dc")
  for k in [-112, -100, -40, 40, 90]:
    _, _, dq, dc = _tc(ops, q, c, inv_t, w, g=2.0 ** k)
    _assert_scaled_bits(dq, dq0, k, f"grad_loss 2^{k} dq")
    _assert_scaled_bits(dc, dc0, k, f"grad_loss 2^{k} dc")


@gpu
@pytest.mark.parametrize("g", [2.0 ** -112, -(2.0 ** -100)])
def test_tiny_grad_loss(ops, sms, g):
  """grad_loss below 2^-98 with ordinary embeddings: the dq factor is not a normal number, the gradients are."""
  B, C = 1024, 1024
  q, c = _pairs(B, C, 64, 241)
  w = torch.rand(B, generator=_gen(242), device="cuda") + 0.5
  _verify(ops, sms, f"grad_loss {g:.3g}", q, c, 1.3, w, g=g)


def _ws_sentinel(nbytes):
  return torch.full((_cdiv(nbytes, 4),), SENTINEL, dtype=torch.int32, device="cuda")


def _sentinel(n):
  return torch.full((n,), SENTINEL, dtype=torch.int32, device="cuda").view(torch.float32)


def _raw_fwd(ops, q, c, inv_t, w, bias, ids, mask):
  B, d = q.shape; C = c.shape[0]
  ws = _ws_sentinel(ops.lib().tfrs_inbatch_softmax_tc_workspace_bytes(B, C, d, int(ids is not None), int(mask is not None)))
  loss, lse = _sentinel(1), _sentinel(B)
  ops.check(ops.lib().tfrs_inbatch_softmax_tc_fwd(ops.ptr(q), ops.ptr(c), B, C, d, ops.c_f(inv_t), ops.ptr(w), ops.ptr(bias),
                                                  ops.ptr(ids), ops.ptr(mask), ops.ptr(loss), ops.ptr(lse),
                                                  ctypes.c_void_p(ws.data_ptr()), ws.numel() * 4, ops.stream()), "tc_fwd")
  return loss.view(()), lse


def _raw_bwd(ops, q, c, lse, inv_t, w, bias, ids, mask, g):
  B, d = q.shape; C = c.shape[0]
  ws = _ws_sentinel(ops.lib().tfrs_inbatch_softmax_tc_bwd_workspace_bytes(B, C, d, int(ids is not None), int(mask is not None)))
  dq, dc = _sentinel(B * d).view(B, d), _sentinel(C * d).view(C, d)
  ops.check(ops.lib().tfrs_inbatch_softmax_tc_bwd(ops.ptr(q), ops.ptr(c), B, C, d, ops.c_f(inv_t), ops.ptr(w), ops.ptr(bias),
                                                  ops.ptr(ids), ops.ptr(mask), ops.ptr(lse), ops.ptr(_gl(g)), ops.ptr(dq),
                                                  ops.ptr(dc), ctypes.c_void_p(ws.data_ptr()), ws.numel() * 4, ops.stream()),
            "tc_bwd")
  return dq, dc


@gpu
@pytest.mark.parametrize("B,C,opts", [(512, 16384, False), (600, 777, True), (1025, 16896, False)])
def test_repeat_and_sentinel_workspace(ops, B, C, opts):
  """Two calls give the same bits, and so does a call whose workspace and outputs start as NaN-payload sentinels."""
  q, c = _pairs(B, C, 64, 251)
  w = torch.rand(B, generator=_gen(252), device="cuda") - 0.25
  bias, ids, mask = (_bias(C, 253), _ids(B, C, 254), _mask(B, C, 255)) if opts else (None, None, None)
  runs = [_tc(ops, q, c, 10.0, w, bias, ids, mask, g=0.75) for _ in range(2)]
  loss, lse = _raw_fwd(ops, q, c, 10.0, w, bias, ids, mask)
  dq, dc = _raw_bwd(ops, q, c, runs[0][1], 10.0, w, bias, ids, mask, 0.75)
  runs.append((loss, lse, dq, dc))
  for run in runs[1:]:
    for name, u, v in zip(["loss", "lse", "dq", "dc"], runs[0], run):
      assert torch.equal(_bits(u), _bits(v)), f"{name} differs between calls"


# ------------------------------------------------------------------------------------------------
# 6. The exact kernels with more than one row block
# ------------------------------------------------------------------------------------------------
def _rows_per_block(B, C):
  """softmax.cu sm_rows_per_block: the [rows, C] score block stays within 128 MB."""
  r = max(128, ((128 << 20) // (C * 4)) // 128 * 128)
  return min(r, B)


@gpu
def test_exact_forward_and_backward_multi_block(ops, monkeypatch):
  """d = 160 is beyond the tensor cores: forward and backward run on the exact kernels in row blocks."""
  B, C, d = 2000, 40000, 160
  assert _rows_per_block(B, C) < B
  q, c = _pairs(B, C, d, 261)
  w = torch.rand(B, generator=_gen(262), device="cuda") + 0.5
  spy = _Spy(ops, monkeypatch)
  loss, dq, dc = _autograd(ops, q, c, w, 0.05)
  assert (spy.fwd, spy.bwd) == (0, 0)
  _, lse = _exact_fwd(ops, q, c, 20.0, w)
  r = reference(q, c, 20.0, w, chain=chain_exact(C), rel=(rel_exact(C), rel_exact(B)))
  check_all(r, "exact multi-block", loss, lse, dq, dc)


def _maxsim_reference(q3, c, inv_t, w, chain, rel):
  """float64 maxsim loss: s_ij = max_h q_ih . c_j; the gradient goes to the maximising head(s), split evenly among ties."""
  q64, c64 = q3.double(), c.double()
  B, H, d = q64.shape
  C = c64.shape[0]
  sh = torch.einsum("bhd,cd->bhc", q64, c64)
  s = sh.max(1).values
  at = (sh == s[:, None, :]).double()
  at = at / at.sum(1, keepdim=True)
  l = s * inv_t
  lse = torch.logsumexp(l, 1)
  # every head's bar (E) is below 1e-5 (max_h |q_ih|) . |c_j|; the scores themselves are exact here
  E = 1e-5 * abs(inv_t) * (q64.abs().amax(1) @ c64.abs().T) + 2.0 ** -22 * l.abs()
  eps = 2.0 ** -21 * chain + 2.0 ** -19 + 2.0 ** -22 * (lse.abs() + 1) + C * 2.0 ** -126
  barL = E.max(1).values + eps
  eye = torch.eye(B, C, dtype=F64, device=q3.device)
  w64 = w.double()
  loss = float((w64 * (lse - l.diagonal())).sum())
  bar_loss = float((w64.abs() * (barL + E.diagonal()) + 2.0 ** -21 * (w64 * (lse - l.diagonal())).abs()).sum())
  p = torch.exp(l - lse[:, None])
  fac = w64 * inv_t
  G = (p - eye) * fac[:, None]
  dP = p * (torch.expm1(E + 2.0 ** -22 * (lse.abs()[:, None] + 10) + barL[:, None]) + 2.0 ** -21)
  Gh = G[:, None, :] * at                                  # [B, H, C]
  dPh = dP[:, None, :] * at * fac.abs()[:, None, None]
  dq = torch.einsum("bhc,cd->bhd", Gh, c64)
  bar_dq = torch.einsum("bhc,cd->bhd", dPh + rel[0] * Gh.abs(), c64.abs())
  dc = torch.einsum("bhc,bhd->cd", Gh, q64)
  bar_dc = torch.einsum("bhc,bhd->cd", dPh + rel[1] * Gh.abs(), q64.abs())
  floor = 2.0 ** -36 * (float(Gh.abs().max()) * c64.abs().sum() + float(c64.abs().max()) * Gh.abs().sum())
  return loss, bar_loss, lse, barL, dq, bar_dq + floor, dc, bar_dc + floor


@gpu
def test_exact_maxsim_multi_block(ops):
  """Multi-head queries with B H above the rows of one score block, on integer data (every score exact in fp32, so the
  maximising heads are the same as in float64), heads 0 and 1 equal for every other query (exact ties)."""
  B, H, C, d = 400, 4, 40000, 32
  assert _rows_per_block(B * H, C) < B * H
  q3 = torch.randint(-3, 4, (B, H, d), generator=_gen(271), device="cuda").float()
  q3[::2, 1] = q3[::2, 0]
  c = torch.randint(-3, 4, (C, d), generator=_gen(272), device="cuda").float()
  w = torch.rand(B, generator=_gen(273), device="cuda") + 0.5
  inv_t = 1.0 / 16
  loss = torch.empty((1,), device="cuda"); lse = torch.empty((B,), device="cuda")
  dq = torch.empty_like(q3); dc = torch.empty_like(c)
  lib = ops.lib()
  ws = torch.empty(lib.tfrs_inbatch_softmax_maxsim_workspace_bytes(B, H, C, d), dtype=torch.uint8, device="cuda")
  ops.check(lib.tfrs_inbatch_softmax_maxsim_fwd(ops.ptr(q3), ops.ptr(c), B, H, C, d, ops.c_f(inv_t), ops.ptr(w), ops.ptr(loss),
                                                ops.ptr(lse), ops.ptr(ws), ws.numel(), ops.stream()), "maxsim_fwd")
  ops.check(lib.tfrs_inbatch_softmax_maxsim_bwd(ops.ptr(q3), ops.ptr(c), B, H, C, d, ops.c_f(inv_t), ops.ptr(w), ops.ptr(lse),
                                                None, ops.ptr(dq), ops.ptr(dc), ops.ptr(ws), ws.numel(), ops.stream()),
            "maxsim_bwd")
  rl, rbl, rlse, rbarL, rdq, rbdq, rdc, rbdc = _maxsim_reference(q3, c, inv_t, w, chain_exact(C),
                                                                  (rel_exact(C), rel_exact(B * H)))
  check(lse, rlse, rbarL, "maxsim (L)")
  check(torch.tensor(float(loss), dtype=F64), torch.tensor(rl, dtype=F64), torch.tensor(rbl, dtype=F64), "maxsim loss")
  check(dq, rdq, rbdq, "maxsim dq (G)")
  check(dc, rdc, rbdc, "maxsim dc (G)")
  assert not torch.equal(dq[::2, 0], torch.zeros_like(dq[::2, 0])) and torch.equal(_bits(dq[::2, 0]), _bits(dq[::2, 1])), \
      "tied heads do not share the gradient evenly"


# ------------------------------------------------------------------------------------------------
# Temperatures the tensor cores do not take
# ------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("B", [511, 512])
def test_negative_temperature(ops, monkeypatch, B):
  """A negative temperature is a valid (order-reversing) scale of the logits: both sides of B = 512 run the exact path."""
  import recommenders_b200 as tfrs
  C = 640
  q, c = _pairs(B, C, 48, 281)
  w = torch.rand(B, generator=_gen(282), device="cuda") + 0.5
  spy = _Spy(ops, monkeypatch)
  loss, dq, dc = _autograd(ops, q, c, w, -0.5)
  assert (spy.fwd, spy.bwd) == (0, 0)
  r = reference(q, c, -2.0, w, chain=chain_exact(C), rel=(rel_exact(C), rel_exact(B)))
  check_all(r, f"T=-0.5 B={B}", loss, None, dq, dc)
  task_loss = tfrs.tasks.Retrieval(temperature=-0.5)(q, c, w, compute_metrics=False)
  check_all(r, f"Retrieval T=-0.5 B={B}", task_loss)


@gpu
def test_options_outside_the_fused_range(ops):
  """Options need the tensor-core forward and backward (B >= 512, d <= 64, T > 0): ops.inbatch_softmax_loss says so, and
  tasks.Retrieval computes them on the score matrix instead -- equal to the float64 oracle."""
  import recommenders_b200 as tfrs
  from oracle import oracle as orc
  B, C = 512, 640
  q, c = _pairs(B, C, 96, 291)
  bias = _bias(C, 292)
  with pytest.raises(NotImplementedError, match="tensor-core path"):
    ops.inbatch_softmax_loss(q, c, None, 0.5, bias)
  q48, c48 = q[:, :48].contiguous(), c[:, :48].contiguous()
  with pytest.raises(NotImplementedError, match="temperature"):
    ops.inbatch_softmax_loss(q48, c48, None, -0.5, bias)
  prob = torch.exp(-bias)
  ids = _ids(B, C, 293)
  for qq, cc, T in [(q, c, 0.5), (q48, c48, -0.5)]:
    qg, cg = qq.clone().requires_grad_(True), cc.clone().requires_grad_(True)
    loss = tfrs.tasks.Retrieval(temperature=T, remove_accidental_hits=True)(
        qg, cg, candidate_sampling_probability=prob, candidate_ids=ids, compute_metrics=False)
    loss.backward()
    el, edq, edc = orc.retrieval_loss_and_grads_general(
        qq.cpu().numpy(), cc.cpu().numpy(), temperature=T, candidate_sampling_probability=prob.cpu().numpy(),
        candidate_ids=ids.cpu().numpy(), remove_accidental_hits_=True)
    loss = float(loss.detach())
    assert abs(loss - el) <= 1e-5 * abs(el), (loss, el)
    for got, ref, name in [(qg.grad, edq, "dq"), (cg.grad, edc, "dc")]:
      err = np.abs(got.detach().cpu().numpy().astype(np.float64) - ref).max()
      assert err <= 1e-5 * np.abs(ref).max(), f"d={qq.shape[1]} T={T} {name}: {err:.3e}"
