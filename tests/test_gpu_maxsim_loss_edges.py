"""The multi-head (maxsim) in-batch softmax loss of tasks.Retrieval on every route a [B, H, d] query takes, and the K3 maxsim
kernels (csrc/softmax.cu sm_row_lse_maxsim, sm_make_grad_maxsim) through the C ABI.

tasks.Retrieval scores candidate j for query i by s_ij = max_h q_ih . c_j (retrieval.py:172-176).  The default loss with a
positive temperature and no option runs in the fused maxsim kernels.  Everything else -- a temperature <= 0, a sampling
probability, accidental-hit removal, a score mask, hard negatives, a custom loss -- takes the maximum over the head rows of
the exact score matrix and follows the reference's op sequence; batch metrics read that score matrix next to the fused
loss.  On every route the gradient of a score goes to the head(s) that attain the maximum, split evenly among exact ties,
as tf.reduce_max's gradient is.

The reference is test_gpu_softmax_tc_edges._maxsim_reference: float64 on the device, one function for every route, with
the bars of that file's exact path.  The scores are fp32 FMA chains of length d (1e-5 of |q| |c| covers d <= 167), the
softmax steps a chain of chain_exact(C), dq an FMA chain of length C and dc one of length B H (rel_exact).  The bars are per
element: a gradient sent to the wrong head misses them on the smallest entry.
Tie data: integer q and c in [-3, 3], so that every score is exact in fp32 and an fp32 tie is a float64 tie; heads 0 and 1
are equal for every other query.  With `distinct`, component 0 of every head is 1 and component 0 of candidate j is
j 2^-10: each row's candidate scores are then distinct (the hard-negative selection is unambiguous) and still exact.
The GPU tests are marked one by one; the bar self-tests at the top run without a GPU.
"""
import math

import numpy as np
import pytest
import torch

from test_gpu_softmax_tc_edges import (F64, FLT_MIN, MIN_FLOAT, SENTINEL, _bits, _cdiv, _gen, _maxsim_reference, _pairs,
                                       _rows_per_block, chain_exact, check, reference, rel_exact)

gpu = pytest.mark.gpu

SM_DQ_SPLITS = 8          # softmax.cu: dq = G . c runs as a split-K SGEMM of this many ranges
T_TIE = 8.0               # a power of two: s / T of the tie data is exact too


def _align(n):
  return _cdiv(n, 256) * 256


def _queries_per_block(B, H, C):
  """softmax.cu smx_queries_per_block: queries whose H head rows share one score block; at least one query."""
  return min(B, max(1, _rows_per_block(B * H, C) // H))


def _int_data(B, H, C, d, seed, distinct=False, device="cuda"):
  """Integer queries [B, H, d] and candidates [C, d] in [-3, 3]; heads 0 and 1 equal for every other query."""
  g = torch.Generator(device=device).manual_seed(seed)
  q3 = torch.randint(-3, 4, (B, H, d), generator=g, device=device).float()
  c = torch.randint(-3, 4, (C, d), generator=g, device=device).float()
  if H > 1:
    q3[::2, 1] = q3[::2, 0]
  if distinct:
    assert C <= 1024
    q3[:, :, 0] = 1.0
    c[:, 0] = torch.arange(C, device=device) * 2.0 ** -10
  return q3.contiguous(), c.contiguous()


def _bars(B, H, C):
  return dict(chain=chain_exact(C), rel=(rel_exact(C), rel_exact(B * H)))


def _check_all(r, what, loss=None, lse=None, dq=None, dc=None):
  rl, rbl, rlse, rbarL, rdq, rbdq, rdc, rbdc = r[:8]
  if loss is not None:
    check(torch.tensor(float(loss), dtype=F64), torch.tensor(rl, dtype=F64), torch.tensor(rbl, dtype=F64), f"{what} loss")
  if lse is not None:
    check(lse, rlse, rbarL, f"{what} lse")
  if dq is not None:
    check(dq, rdq, rbdq, f"{what} dq")
  if dc is not None:
    check(dc, rdc, rbdc, f"{what} dc")


# ------------------------------------------------------------------------------------------------
# The bars have teeth (no GPU): they accept the float64 answer rounded to fp32 and reject planted defects
# ------------------------------------------------------------------------------------------------
def _cpu_options(B, C, seed):
  g = torch.Generator().manual_seed(seed)
  p = torch.exp2(-20 * torch.rand(C, generator=g)); p[::11] = 1.0; p[5::13] = 1e-9
  mask = torch.rand((B, C), generator=g) > 0.2
  mask[3, 3] = False
  return {"bias": -torch.log(torch.clamp(p.double(), 1e-6, 1.0)), "ids": torch.randint(0, 11, (C,), generator=g),
          "mask": mask}


@pytest.mark.parametrize("opts", ["none", "options", "hard"])
def test_bars_accept_the_rounded_float64_answer(opts):
  B, H, C, d = 24, 3, 40, 16
  q3, c = _int_data(B, H, C, d, 1, distinct=opts == "hard", device="cpu")
  w = torch.rand(B, generator=torch.Generator().manual_seed(2)) + 0.5
  kw = {"options": _cpu_options(B, C, 3), "hard": {"hard": 4}}.get(opts, {})
  r = _maxsim_reference(q3, c, 1 / T_TIE, w, g=0.75, **_bars(B, H, C), **kw)
  _check_all(r, f"rounded float64 ({opts})", np.float32(r[0]), r[2].float(), r[4].float(), r[6].float())


def test_bars_reject_a_gradient_given_wholly_to_one_tied_head():
  B, H, C, d = 24, 3, 40, 16
  q3, c = _int_data(B, H, C, d, 4, device="cpu")
  r = _maxsim_reference(q3, c, 1 / T_TIE, None, **_bars(B, H, C))
  dq = r[4].clone()
  dq[::2, 0] += dq[::2, 1]
  dq[::2, 1] = 0
  with pytest.raises(AssertionError, match="dq"):
    check(dq.float(), r[4], r[5], "dq with the tied gradient on head 0")


def test_bars_reject_a_dropped_head():
  B, H, C, d = 24, 3, 40, 16
  q3, c = _int_data(B, H, C, d, 5, device="cpu")
  r = _maxsim_reference(q3, c, 1 / T_TIE, None, **_bars(B, H, C), keep_g=True)
  Gh = r[8].clone()
  Gh[:, H - 1] = 0
  with pytest.raises(AssertionError, match="dc"):
    check(torch.einsum("bhc,bhd->cd", Gh, q3.double()).float(), r[6], r[7], "dc without the last head")


def test_bars_reject_an_unmasked_accidental_hit():
  """One duplicate id: the candidate j >= B of largest probability shares the id of the query it is most probable for."""
  B, H, C, d = 24, 3, 40, 16
  q3, c = _int_data(B, H, C, d, 6, device="cpu")
  r0 = _maxsim_reference(q3, c, 1 / T_TIE, None, **_bars(B, H, C))
  l = torch.einsum("bhd,cd->bhc", q3.double(), c.double()).amax(1) / T_TIE - r0[2][:, None]
  i, j = (int(v) for v in divmod(int(l[:, B:].argmax()), C - B))
  ids = torch.arange(C)
  ids[B + j] = i
  r = _maxsim_reference(q3, c, 1 / T_TIE, None, **_bars(B, H, C), ids=ids)
  with pytest.raises(AssertionError, match="dq"):
    check(r0[4].float(), r[4], r[5], "dq with the hit left in")


def test_one_head_reference_is_the_2d_reference():
  """At H = 1 the options of _maxsim_reference compute what the 2-D reference does (float64 values, not bars)."""
  B, C, d = 30, 50, 8
  g = torch.Generator().manual_seed(7)
  q, c = torch.randn((B, d), generator=g), torch.randn((C, d), generator=g)
  w = torch.rand(B, generator=g) - 0.25
  o = _cpu_options(B, C, 8)
  r3 = _maxsim_reference(q[:, None], c, 0.5, w, g=-1.5, chain=1, rel=(1e-5, 1e-5), **o)
  r2 = reference(q, c, 0.5, w, o["bias"], o["ids"], o["mask"], g=-1.5)
  assert abs(r3[0] - r2.loss) <= 1e-12 * abs(r2.loss)
  for got, want in [(r3[2], r2.lse), (r3[4][:, 0], r2.dq), (r3[6], r2.dc)]:
    torch.testing.assert_close(got, want, rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("B,H,C,d,Rq,blocks", [(340, 3, 65536, 16, 170, 2), (341, 3, 65536, 16, 170, 3),
                                                (3, 129, 262144, 8, 1, 3), (300, 4, 40000, 32, 192, 2),
                                                (300, 1, 40000, 32, 300, 1), (7, 2, 8, 5, 7, 1)])
def test_workspace_restates_the_query_blocks(B, H, C, d, Rq, blocks):
  """The workspace holds one block of Rq H score rows, the row losses and the dq split-K ranges: the restatement of the
  query blocks the GPU cases are named for is the one the library sizes its workspace by."""
  from recommenders_b200 import ops
  assert (_queries_per_block(B, H, C), _cdiv(B, _queries_per_block(B, H, C))) == (Rq, blocks)
  R = Rq * H
  want = _align(R * C * 4) + _align(B * 4) + _align(SM_DQ_SPLITS * R * d * 4)
  assert ops.lib().tfrs_inbatch_softmax_maxsim_workspace_bytes(B, H, C, d) == want


# ------------------------------------------------------------------------------------------------
# tasks.Retrieval on 3-D queries
# ------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def ops():
  from recommenders_b200 import ops as o
  return o


class _Routes:
  """Counts the calls of the fused maxsim loss and of the score matrix."""

  def __init__(self, ops, monkeypatch):
    self.fused = self.scores = 0
    f0, s0 = ops.inbatch_softmax_maxsim_loss, ops.scores

    def fused(*a, **k):
      self.fused += 1
      return f0(*a, **k)

    def scores(*a, **k):
      self.scores += 1
      return s0(*a, **k)
    monkeypatch.setattr(ops, "inbatch_softmax_maxsim_loss", fused)
    monkeypatch.setattr(ops, "scores", scores)


def _custom_loss(y_true, y_pred, sample_weight=None):
  """Categorical cross-entropy from logits, reduction SUM, through torch's cross_entropy."""
  per = torch.nn.functional.cross_entropy(y_pred, y_true, reduction="none")
  if sample_weight is not None:
    per = per * sample_weight.reshape(-1)
  return per.sum()


def _route(route, B, C, seed):
  """(Retrieval arguments, call arguments, reference options, temperature) of a route."""
  task, call, ref, T = {}, {}, {}, T_TIE
  if route == "T=-0.5":
    T = -0.5
  elif route == "sampling":
    p = torch.exp2(-24 * torch.rand(C, generator=_gen(seed), device="cuda"))
    p[::11] = 1.0                                          # no correction
    p[5::13] = 1e-9                                        # below the 1e-6 clip
    call["candidate_sampling_probability"] = p
    ref["bias"] = -torch.log(torch.clamp(p.double(), 1e-6, 1.0))
  elif route == "hits":
    ids = torch.randint(0, 9, (C,), generator=_gen(seed), device="cuda")
    task["remove_accidental_hits"] = True
    call["candidate_ids"] = ref["ids"] = ids
  elif route == "mask":
    m = torch.rand((B, C), generator=_gen(seed), device="cuda") > 0.3
    m[:, 7] = False                                        # a column masked for every row (a positive among them)
    m[3, 3] = False                                        # another masked positive
    call["score_mask"] = ref["mask"] = m
  elif route.startswith("hard"):
    n = C - 1 if route == "hard C-1" else int(route[4:])
    task["num_hard_negatives"] = ref["hard"] = n
  elif route == "custom":
    task["loss"] = _custom_loss
  elif route == "metrics":
    from recommenders_b200 import metrics
    task["batch_metrics"] = [metrics.TopKCategoricalAccuracy(k=20, name="acc20")]
    task["loss_metrics"] = [metrics.Mean("loss")]
  task["temperature"] = T
  return task, call, ref, T


ROUTES = ["fused", "T=-0.5", "sampling", "hits", "mask", "hard1", "hard4", "hard C-1", "custom", "metrics"]


def _task_run(ops, monkeypatch, q3, c, w, task_kw, call_kw):
  import recommenders_b200 as tfrs
  routes = _Routes(ops, monkeypatch)
  task = tfrs.tasks.Retrieval(**task_kw)
  qg, cg = q3.clone().requires_grad_(True), c.clone().requires_grad_(True)
  loss = task(qg, cg, sample_weight=w, **call_kw)
  loss.backward()
  return task, routes, loss.detach(), qg.grad, cg.grad


@gpu
@pytest.mark.parametrize("wshape", ["B", "B,1"])
@pytest.mark.parametrize("H", [1, 2, 3, 8])
@pytest.mark.parametrize("route", ROUTES)
def test_every_route(ops, monkeypatch, route, H, wshape):
  """Loss, dq and dc of loss.backward() per element, the route taken, and on the metrics route TopKCategoricalAccuracy of
  the maxsim scores and the loss the loss metric receives."""
  B, C, d = 40, 72, 16
  q3, c = _int_data(B, H, C, d, 11 + H, distinct=True)
  w = torch.rand(B, generator=_gen(12), device="cuda") + 0.5
  task_kw, call_kw, ref_kw, T = _route(route, B, C, 13)
  task, routes, loss, dq, dc = _task_run(ops, monkeypatch, q3, c, w if wshape == "B" else w[:, None], task_kw, call_kw)
  fused = route in ("fused", "metrics")
  assert (routes.fused, routes.scores) == (int(fused), int(not fused or route == "metrics")), route
  r = _maxsim_reference(q3, c, 1.0 / T, w, **_bars(B, H, C), **ref_kw)
  _check_all(r, f"{route} H={H} w[{wshape}]", loss, None, dq, dc)
  if route == "metrics":
    s = torch.einsum("bhd,cd->bhc", q3.double(), c.double()).amax(1)
    hit = ((s > s.diagonal()[:, None]).sum(1) < 20).double()
    want = float((hit * w.double()).sum() / w.double().sum())
    assert 0 < float(hit.mean()) < 1, "the accuracy premise: some rows in the top 20, some not"
    acc, mean = task.metrics
    assert abs(acc.result() - want) <= 1e-12, (acc.result(), want)
    assert mean.result() == float(loss)


@gpu
@pytest.mark.parametrize("H", [2, 3, 8])
@pytest.mark.parametrize("route", ["mask", "custom", "T=-0.5", "hard C-1"])
def test_tied_heads_split_the_gradient(ops, monkeypatch, route, H):
  """Heads 0 and 1 are equal for every other query.  On the score-matrix route each of the two gets half the gradient of
  their score: the same bits, nonzero, equal to half the float64 total -- as tf.reduce_max and the fused kernels split it."""
  B, C, d = 40, 72, 16
  q3, c = _int_data(B, H, C, d, 21 + H, distinct=True)
  w = torch.rand(B, generator=_gen(22), device="cuda") + 0.5
  task_kw, call_kw, ref_kw, T = _route(route, B, C, 23)
  if route == "mask":
    call_kw["score_mask"] = ref_kw["mask"] = torch.ones((B, C), dtype=torch.bool, device="cuda")
  _, routes, _, dq, _ = _task_run(ops, monkeypatch, q3, c, w, task_kw, call_kw)
  assert routes.fused == 0 and routes.scores == 1
  h0, h1 = _bits(dq[::2, 0]), _bits(dq[::2, 1])
  differ = (h0 != h1).any(1)
  if bool(differ.any()):
    b = 2 * int(torch.nonzero(differ)[0])
    raise AssertionError(f"{route} H={H}: query {b} has tied heads 0 and 1 (equal queries), but they get different "
                         f"gradients: |dq| sums {float(dq[b, 0].abs().sum()):.6g} and {float(dq[b, 1].abs().sum()):.6g}; "
                         f"{int(differ.sum())} of {differ.numel()} tied queries differ")
  zero = (dq[::2, 0] == 0).all(1)
  assert not bool(zero.any()), f"{route} H={H}: query {2 * int(torch.nonzero(zero)[0])} has no gradient on its tied heads"
  r = _maxsim_reference(q3, c, 1.0 / T, w, **_bars(B, H, C), **ref_kw)
  half = 0.5 * (r[4][::2, 0] + r[4][::2, 1])
  for h in (0, 1):
    check(dq[::2, h], half, r[5][::2, h], f"{route} H={H} tied head {h}: half the tied gradient")


@gpu
@pytest.mark.parametrize("T", [T_TIE, 5.0])
@pytest.mark.parametrize("H", [1, 3, 8])
@pytest.mark.parametrize("force", ["score_mask", "sampling_probability"])
def test_routes_agree(ops, monkeypatch, force, H, T):
  """An all-true score mask or a sampling probability of all ones changes no logit but forces the score-matrix route: on
  the tie data its loss and gradients agree with the fused route's within both routes' bars.  1/5 is not an fp32 number:
  the fused kernels multiply by its rounding, the score-matrix route divides by 5."""
  B, C, d = 64, 100, 16
  q3, c = _int_data(B, H, C, d, 31 + H)
  w = torch.rand(B, generator=_gen(33), device="cuda") + 0.5
  force_kw = {"score_mask": torch.ones((B, C), dtype=torch.bool, device="cuda")} if force == "score_mask" else \
      {"candidate_sampling_probability": torch.ones(C, device="cuda")}
  _, routes, *fused = _task_run(ops, monkeypatch, q3, c, w, {"temperature": T}, {})
  assert (routes.fused, routes.scores) == (1, 0)
  _, routes, *matrix = _task_run(ops, monkeypatch, q3, c, w, {"temperature": T}, force_kw)
  assert (routes.fused, routes.scores) == (0, 1)
  r = _maxsim_reference(q3, c, 1.0 / T, w, **_bars(B, H, C))
  what = f"H={H} T={T}"
  _check_all(r, f"fused {what}", fused[0], None, fused[1], fused[2])
  _check_all(r, f"{force} {what}", matrix[0], None, matrix[1], matrix[2])
  check(torch.tensor(float(matrix[0]), dtype=F64), torch.tensor(float(fused[0]), dtype=F64),
        torch.tensor(2 * r[1], dtype=F64), f"{force} vs fused {what} loss")
  check(matrix[1], fused[1].double(), 2 * r[5], f"{force} vs fused {what} dq")
  check(matrix[2], fused[2].double(), 2 * r[7], f"{force} vs fused {what} dc")


# ------------------------------------------------------------------------------------------------
# The K3 maxsim kernels through the C ABI
# ------------------------------------------------------------------------------------------------
def _sentinel(n):
  return torch.full((n,), SENTINEL, dtype=torch.int32, device="cuda").view(torch.float32)


def _gl(g):
  return None if g is None else torch.tensor([g], dtype=torch.float32, device="cuda")


def _abi(ops, q3, c, inv_t, w=None, g=None, sentinel=False):
  """tfrs_inbatch_softmax_maxsim_fwd, then _bwd on its lse: (loss, lse, dq, dc).  With `sentinel` the workspace and the
  outputs start as NaN-payload sentinels, else the workspace starts as zeros."""
  lib = ops.lib()
  B, H, d = q3.shape
  C = c.shape[0]
  nbytes = lib.tfrs_inbatch_softmax_maxsim_workspace_bytes(B, H, C, d)
  ws = _sentinel(_cdiv(nbytes, 4)) if sentinel else torch.zeros(_cdiv(nbytes, 4), device="cuda")
  if sentinel:
    loss, lse, dq, dc = _sentinel(1), _sentinel(B), _sentinel(B * H * d).view(B, H, d), _sentinel(C * d).view(C, d)
  else:
    loss, lse, dq, dc = torch.empty(1, device="cuda"), torch.empty(B, device="cuda"), torch.empty_like(q3), torch.empty_like(c)
  ops.check(lib.tfrs_inbatch_softmax_maxsim_fwd(ops.ptr(q3), ops.ptr(c), B, H, C, d, ops.c_f(inv_t), ops.ptr(w),
                                                ops.ptr(loss), ops.ptr(lse), ops.ptr(ws), nbytes, ops.stream()),
            "maxsim_fwd")
  ops.check(lib.tfrs_inbatch_softmax_maxsim_bwd(ops.ptr(q3), ops.ptr(c), B, H, C, d, ops.c_f(inv_t), ops.ptr(w),
                                                ops.ptr(lse), ops.ptr(_gl(g)), ops.ptr(dq), ops.ptr(dc), ops.ptr(ws), nbytes,
                                                ops.stream()), "maxsim_bwd")
  return loss.view(()), lse, dq, dc


def _abi_2d(ops, q, c, inv_t, w=None, g=None):
  """tfrs_inbatch_softmax_fwd, then _bwd on its lse: (loss, lse, dq, dc)."""
  lib = ops.lib()
  B, d = q.shape
  C = c.shape[0]
  nbytes = lib.tfrs_inbatch_softmax_workspace_bytes(B, C, d)
  ws = torch.zeros(_cdiv(nbytes, 4), device="cuda")
  loss, lse, dq, dc = torch.empty(1, device="cuda"), torch.empty(B, device="cuda"), torch.empty_like(q), torch.empty_like(c)
  ops.check(lib.tfrs_inbatch_softmax_fwd(ops.ptr(q), ops.ptr(c), B, C, d, ops.c_f(inv_t), ops.ptr(w), ops.ptr(loss),
                                         ops.ptr(lse), ops.ptr(ws), nbytes, ops.stream()), "inbatch_softmax_fwd")
  ops.check(lib.tfrs_inbatch_softmax_bwd(ops.ptr(q), ops.ptr(c), B, C, d, ops.c_f(inv_t), ops.ptr(w), ops.ptr(lse),
                                         ops.ptr(_gl(g)), ops.ptr(dq), ops.ptr(dc), ops.ptr(ws), nbytes, ops.stream()),
            "inbatch_softmax_bwd")
  return loss.view(()), lse, dq, dc


def _same_bits(u, v, what):
  diff = _bits(u) != _bits(v)
  assert not bool(diff.any()), f"{what}: {int(diff.sum())} of {diff.numel()} values differ in their bits"


@gpu
@pytest.mark.parametrize("B,C,d", [(1, 1, 8), (300, 1000, 32), (257, 257, 160), (600, 131072, 16)])
def test_one_head_is_the_2d_kernel(ops, B, C, d):
  """H = 1 runs the same fp32 operations as the 2-D exact kernels: loss, lse, dq and dc with the same bits.  The last
  shape has three row blocks."""
  q, c = _pairs(B, C, d, 41)
  w = torch.rand(B, generator=_gen(42), device="cuda") - 0.25
  one = _abi(ops, q[:, None].contiguous(), c, 20.0, w, 0.75)
  flat = _abi_2d(ops, q, c, 20.0, w, 0.75)
  for name, u, v in zip(["loss", "lse", "dq", "dc"], one, flat):
    _same_bits(u.reshape(v.shape), v, f"H=1 vs 2-D B={B} C={C} d={d} {name}")


@gpu
@pytest.mark.parametrize("H", [2, 4, 8])
def test_equal_heads(ops, H):
  """H copies of one head: the loss and lse bits of H = 1, and per head dq(H = 1) / H bit for bit (the even split divides
  by a power of two).  Unit-norm rows at T = 0.05 keep every p above 2^-100, so no G entry is subnormal; H = 4 and 8 run
  two and four row blocks where H = 1 runs one."""
  B, C, d = 300, 40000, 32
  assert [_cdiv(B, _queries_per_block(B, h, C)) for h in (1, 2, 4, 8)] == [1, 1, 2, 4]
  q, c = _pairs(B, C, d, 51)
  w = torch.rand(B, generator=_gen(52), device="cuda") + 0.5
  l = (q.double() @ c.double().T) * 20.0
  assert float((l - torch.logsumexp(l, 1, keepdim=True)).min()) > -100 * math.log(2), "some p is below 2^-100"
  one = _abi(ops, q[:, None].contiguous(), c, 20.0, w, 0.75)
  q3 = q[:, None].expand(B, H, d).contiguous()
  many = _abi(ops, q3, c, 20.0, w, 0.75)
  _same_bits(many[0], one[0], f"H={H} equal heads loss")
  _same_bits(many[1], one[1], f"H={H} equal heads lse")
  dq1 = one[2][:, 0]
  assert bool(((dq1.abs() / H >= FLT_MIN) | (dq1 == 0)).all()), "a dq(H = 1) / H is not a normal number"
  for h in range(H):
    _same_bits(many[2][:, h], dq1 / H, f"H={H} equal heads dq head {h} vs dq(H=1) / {H}")
  r = _maxsim_reference(q3, c, 20.0, w, g=0.75, **_bars(B, H, C))
  check(many[3], r[6], r[7], f"H={H} equal heads dc")


@gpu
@pytest.mark.parametrize("H", [3, 8])
def test_head_permutation(ops, H):
  """Permuting the heads (tied ones among them) permutes the dq rows bit for bit and leaves the loss and lse bits."""
  B, C, d = 200, 3000, 24
  q3, c = _int_data(B, H, C, d, 61 + H)
  w = torch.rand(B, generator=_gen(62), device="cuda") + 0.5
  perm = torch.randperm(H, generator=torch.Generator().manual_seed(63)).cuda()
  assert bool((perm != torch.arange(H, device="cuda")).any())
  a = _abi(ops, q3, c, 1 / T_TIE, w, -1.5)
  b = _abi(ops, q3[:, perm].contiguous(), c, 1 / T_TIE, w, -1.5)
  _same_bits(b[0], a[0], f"H={H} permuted loss")
  _same_bits(b[1], a[1], f"H={H} permuted lse")
  _same_bits(b[2], a[2][:, perm], f"H={H} permuted dq")
  r = _maxsim_reference(q3, c, 1 / T_TIE, w, g=-1.5, **_bars(B, H, C))
  _check_all(r, f"H={H} unpermuted", *a)


@gpu
@pytest.mark.parametrize("B,H,C,d,Rq,blocks", [(340, 3, 65536, 16, 170, 2), (341, 3, 65536, 16, 170, 3),
                                                (3, 129, 262144, 8, 1, 3)])
def test_row_block_edges(ops, B, H, C, d, Rq, blocks):
  """B = 2 Rq (the last block full) and 2 Rq + 1 (a last block of one query), with Rq = 170 queries in a block of 510 of
  its 512 rows; and H = 129 above the 128 rows of a block at C = 2^18, where the block clamps to one query of 129 rows:
  three blocks, and dc accumulates across them."""
  assert (_queries_per_block(B, H, C), _cdiv(B, Rq)) == (Rq, blocks)
  q3, c = _int_data(B, H, C, d, 71)
  w = torch.rand(B, generator=_gen(72), device="cuda") + 0.5
  got = _abi(ops, q3, c, 1 / T_TIE, w, 0.75)
  r = _maxsim_reference(q3, c, 1 / T_TIE, w, g=0.75, **_bars(B, H, C))
  _check_all(r, f"blocks B={B} H={H} C={C}", *got)


@gpu
@pytest.mark.parametrize("B,H,C,d", [(1, 1, 1, 4), (1, 3, 1, 4), (7, 2, 8, 5), (31, 3, 31, 16), (40, 2, 255, 16),
                                     (40, 4, 257, 16), (30, 3, 100, 1), (30, 5, 100, 3), (50, 2, 300, 160)])
def test_small_and_uneven_shapes(ops, B, H, C, d):
  """B = C = 1, C = B + 1, C below and just above one 256-thread stride, d of 1, 3 and 160."""
  q3, c = _int_data(B, H, C, d, 81 + d)
  w = torch.rand(B, generator=_gen(82), device="cuda") + 0.5
  inv_t = 1 / T_TIE if d > 3 else 0.5
  got = _abi(ops, q3, c, inv_t, w, 0.75)
  r = _maxsim_reference(q3, c, inv_t, w, g=0.75, **_bars(B, H, C))
  _check_all(r, f"shape B={B} H={H} C={C} d={d}", *got)


@gpu
@pytest.mark.parametrize("g", [0.0, -1.5, 2.0 ** -20])
def test_weights_and_grad_loss(ops, g):
  """Weights in [-1, 1) with every 7th one 0; grad_loss 0 gives gradients of exactly 0."""
  B, H, C, d = 200, 4, 600, 16
  q3, c = _int_data(B, H, C, d, 91)
  w = torch.rand(B, generator=_gen(92), device="cuda") * 2 - 1
  w[::7] = 0
  got = _abi(ops, q3, c, 1 / T_TIE, w, g)
  r = _maxsim_reference(q3, c, 1 / T_TIE, w, g=g, **_bars(B, H, C))
  _check_all(r, f"weights grad_loss={g:g}", *got)
  if g == 0:
    assert not bool(got[2].any()) and not bool(got[3].any()), "grad_loss 0 leaves a nonzero gradient"


@gpu
@pytest.mark.parametrize("B,H,C,d", [(37, 3, 500, 16), (300, 4, 40000, 32)])
def test_sentinel_workspace_and_repeat(ops, B, H, C, d):
  """Two calls give the same bits, and so does a call whose workspace and outputs start as NaN-payload sentinels."""
  q3, c = _int_data(B, H, C, d, 101)
  w = torch.rand(B, generator=_gen(102), device="cuda") - 0.25
  runs = [_abi(ops, q3, c, 1 / T_TIE, w, 0.5), _abi(ops, q3, c, 1 / T_TIE, w, 0.5),
          _abi(ops, q3, c, 1 / T_TIE, w, 0.5, sentinel=True)]
  for k, run in enumerate(runs[1:], 1):
    for name, u, v in zip(["loss", "lse", "dq", "dc"], runs[0], run):
      _same_bits(v, u, f"call {k} {name}")


@gpu
@pytest.mark.parametrize("case", ["C < B", "H = 0", "B H = 2^31", "workspace too small", "no workspace"])
def test_argument_errors(ops, case):
  """Each bad call returns its error before any launch and writes nothing.  B H = 2^31 is an argument check only: the
  buffers passed are a few floats that no kernel may touch."""
  from recommenders_b200 import _ffi
  lib = ops.lib()
  B, H, C, d = 4, 2, 8, 4
  if case == "C < B":
    C = 3
  elif case == "H = 0":
    H = 0
  elif case == "B H = 2^31":
    B, H, C, d = 1 << 16, 1 << 15, 1 << 16, 1
  small = case in ("C < B", "H = 0", "B H = 2^31")
  nbytes = 256 if small else lib.tfrs_inbatch_softmax_maxsim_workspace_bytes(B, H, C, d)
  ws = None if case == "no workspace" else _sentinel(_cdiv(nbytes, 4))
  if case == "workspace too small":
    nbytes -= 1
  code, msg = ((-1, "too large") if case == "B H = 2^31" else (-1, "bad arguments")) if small else \
      (-4, "workspace too small")
  bufs = [_sentinel(64) for _ in range(6)]
  q3, c, loss, lse, dq, dc = bufs
  w = torch.ones(8, device="cuda")
  torch.cuda.synchronize()
  n0 = lib.tfrs_launch_count()
  calls = {
      "fwd": lambda: lib.tfrs_inbatch_softmax_maxsim_fwd(ops.ptr(q3), ops.ptr(c), B, H, C, d, ops.c_f(1.0), ops.ptr(w),
                                                         ops.ptr(loss), ops.ptr(lse), ops.ptr(ws), nbytes, ops.stream()),
      "bwd": lambda: lib.tfrs_inbatch_softmax_maxsim_bwd(ops.ptr(q3), ops.ptr(c), B, H, C, d, ops.c_f(1.0), ops.ptr(w),
                                                         ops.ptr(lse), None, ops.ptr(dq), ops.ptr(dc), ops.ptr(ws), nbytes,
                                                         ops.stream())}
  for name, call in calls.items():
    rc = call()
    assert rc == code and msg in _ffi.last_error(), f"{case} {name}: code {rc}, {_ffi.last_error()!r}"
  assert lib.tfrs_launch_count() == n0, f"{case}: a kernel was launched"
  torch.cuda.synchronize()
  for t in bufs + ([] if ws is None else [ws]):
    assert bool((t.view(torch.int32) == SENTINEL).all()), f"{case}: a buffer was written"
