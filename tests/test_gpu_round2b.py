"""Round-2 (second half) GPU parity tests, through the C ABI: the remaining Retrieval loss options fused into the
tensor-core loss (accidental-hit removal, score_mask), hard-negative mining on the top-K scan, the general tensor-core
GEMM, the low-rank Cross / MultiLayerDCN on tensor cores, hot-row staging in the gather.  The checker is the float64
oracle (oracle/oracle.py); bars are written next to each comparison."""
import numpy as np
import pytest
import torch

from oracle import oracle as orc

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ops():
  from recommenders_b200 import ops as o
  return o


def _rand(shape, seed, scale=1.0):
  g = torch.Generator(device="cuda"); g.manual_seed(seed)
  return torch.randn(shape, generator=g, device="cuda") * scale


def _close(got, ref, rel, what):
  ref = np.asarray(ref, np.float64); got = np.asarray(got, np.float64)
  scale = np.abs(ref).max()
  err = np.abs(got - ref).max()
  assert err <= rel * scale, f"{what}: max err {err:.3e} vs scale {scale:.3e} (bar {rel:g} relative)"


# ------------------------------------------------------------------------------------------------
# Retrieval loss options inside the tensor-core loss (tasks/retrieval.py:187-203, layers/loss.py:114-158)
# ------------------------------------------------------------------------------------------------
def _loss_case(B, C, d, seed, scale):
  q = _rand((B, d), seed, scale); c = _rand((C, d), seed + 1, scale)
  g = torch.Generator(device="cuda"); g.manual_seed(seed + 2)
  ids = torch.randint(0, max(B // 3, 2), (C,), generator=g, device="cuda", dtype=torch.int64)   # many duplicate ids
  ids[::5] += 1 << 33                                                                            # exercise the high word
  mask = torch.rand((B, C), generator=g, device="cuda") < 0.85
  mask[torch.arange(B), torch.arange(B)] = True                                                  # positives stay visible
  prob = torch.rand((C,), generator=g, device="cuda") * 0.5 + 1e-3
  w = torch.rand((B,), generator=g, device="cuda") + 0.5
  return q, c, ids, mask, prob, w


@pytest.mark.parametrize("B,C,d", [(512, 512, 64), (1024, 1536, 32), (640, 1000, 64)])
@pytest.mark.parametrize("opts", ["ids", "mask", "ids+mask+bias+temp+w"])
def test_loss_options_fused_forward_backward(ops, B, C, d, opts):
  q, c, ids, mask, prob, w = _loss_case(B, C, d, 11, 0.4)
  use_ids = "ids" in opts; use_mask = "mask" in opts; use_bias = "bias" in opts
  temp = 0.7 if "temp" in opts else None
  sw = w if "+w" in opts else None
  bias = -torch.log(torch.clamp(prob, 1e-6, 1.0)) if use_bias else None
  qg = q.clone().requires_grad_(True); cg = c.clone().requires_grad_(True)
  loss = ops.inbatch_softmax_loss(qg, cg, sw, temp, bias, ids if use_ids else None, mask if use_mask else None)
  (loss * 1.5).backward()
  rl, rdq, rdc = orc.retrieval_loss_and_grads_general(
      q.cpu().numpy(), c.cpu().numpy(), None if sw is None else sw.cpu().numpy(), temp,
      prob.cpu().numpy() if use_bias else None, ids.cpu().numpy(), use_ids, mask.cpu().numpy() if use_mask else None)
  assert abs(float(loss) - rl) <= 1e-5 * abs(rl), (float(loss), rl)     # bar: 1e-5 relative (north_star)
  _close(qg.grad.cpu().numpy(), 1.5 * rdq, 1e-5, "dq")
  _close(cg.grad.cpu().numpy(), 1.5 * rdc, 1e-5, "dc")


def test_score_mask_degenerate_rows(ops):
  """A fully masked row (every logit MIN_FLOAT -> loss log C, zero gradient) and a row whose only visible entry is the
  positive (loss 0)."""
  B = C = 512; d = 64
  q, c, ids, mask, prob, w = _loss_case(B, C, d, 21, 0.3)
  mask[5, :] = False
  mask[9, :] = False; mask[9, 9] = True
  qg = q.clone().requires_grad_(True); cg = c.clone().requires_grad_(True)
  loss = ops.inbatch_softmax_loss(qg, cg, None, None, None, None, mask)
  loss.backward()
  rl, rdq, rdc = orc.retrieval_loss_and_grads_general(q.cpu().numpy(), c.cpu().numpy(), score_mask=mask.cpu().numpy())
  # row 5 of the reference: lse - pos with both ~MIN_FLOAT; the max-subtracted form gives exactly log(C)
  assert abs(float(loss) - rl) <= 1e-5 * abs(rl), (float(loss), rl)
  assert float(qg.grad[5].abs().max()) == 0.0 and float(qg.grad[9].abs().max()) <= 1e-5
  _close(qg.grad.cpu().numpy(), rdq, 1e-5, "dq")
  _close(cg.grad.cpu().numpy(), rdc, 1e-5, "dc")


def test_retrieval_task_routes_options_to_the_fused_kernels(ops, monkeypatch):
  """tfrs.tasks.Retrieval with remove_accidental_hits / score_mask / sampling probability never builds the [B,C] matrix."""
  import recommenders_b200 as tfrs
  B, C, d = 768, 1024, 64
  q, c, ids, mask, prob, w = _loss_case(B, C, d, 31, 0.4)
  monkeypatch.setattr(ops, "scores", lambda *a, **k: (_ for _ in ()).throw(AssertionError("logits were materialised")))
  task = tfrs.tasks.Retrieval(temperature=0.5, remove_accidental_hits=True)
  qg = q.clone().requires_grad_(True); cg = c.clone().requires_grad_(True)
  loss = task(qg, cg, sample_weight=w, candidate_sampling_probability=prob, candidate_ids=ids, score_mask=mask,
              compute_metrics=False)
  loss.backward()
  rl, rdq, rdc = orc.retrieval_loss_and_grads_general(q.cpu().numpy(), c.cpu().numpy(), w.cpu().numpy(), 0.5, prob.cpu().numpy(),
                                                     ids.cpu().numpy(), True, mask.cpu().numpy())
  assert abs(float(loss) - rl) <= 1e-5 * abs(rl)
  _close(qg.grad.cpu().numpy(), rdq, 1e-5, "dq"); _close(cg.grad.cpu().numpy(), rdc, 1e-5, "dc")
  # string ids (the reference's tests use them) are factorised on the host: same result
  sid = np.asarray([f"id{int(v)}" for v in ids.cpu().numpy()])
  loss2 = task(q, c, sample_weight=w, candidate_sampling_probability=prob, candidate_ids=sid, score_mask=mask, compute_metrics=False)
  assert float(loss2) == float(loss)
  with pytest.raises(ValueError):
    task(q, c, compute_metrics=False)   # accidental-hit removal without ids (retrieval.py:194-199)


def test_loss_options_match_the_materialised_reference_sequence(ops):
  """Same numbers as the reference's op sequence on the exact score matrix (oracle.retrieval_loss, float32 logits)."""
  B, C, d = 512, 700, 64
  q, c, ids, mask, prob, w = _loss_case(B, C, d, 41, 0.5)
  loss = ops.inbatch_softmax_loss(q, c, w, 2.0, -torch.log(torch.clamp(prob, 1e-6, 1.0)), ids, mask)
  ref = orc.retrieval_loss(q.cpu().numpy(), c.cpu().numpy(), w.cpu().numpy(), temperature=2.0,
                           candidate_sampling_probability=prob.cpu().numpy(), candidate_ids=ids.cpu().numpy(),
                           remove_accidental_hits_=True, score_mask=mask.cpu().numpy())
  assert abs(float(loss) - ref) <= 1e-5 * abs(ref), (float(loss), ref)


# ------------------------------------------------------------------------------------------------
# hard-negative mining on the top-K scan (tasks/retrieval.py:205-210, layers/loss.py:61-111)
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B,C,d,n,temp,weighted", [(300, 300, 32, 5, None, False), (512, 2048, 64, 10, 0.5, True),
                                                    (1024, 20000, 64, 20, 2.0, True), (64, 40, 16, 100, None, False)])
def test_hard_negative_mining_fused(ops, B, C, d, n, temp, weighted):
  if C < B:
    B = C
  q = _rand((B, d), 51, 0.5); c = _rand((C, d), 52, 0.5)
  w = (torch.rand((B,), device="cuda") + 0.5) if weighted else None
  qg = q.clone().requires_grad_(True); cg = c.clone().requires_grad_(True)
  loss = ops.hard_negative_softmax_loss(qg, cg, n, w, temp)
  loss.backward()
  rl, rdq, rdc = orc.retrieval_loss_and_grads_general(q.cpu().numpy(), c.cpu().numpy(), None if w is None else w.cpu().numpy(),
                                                     temp, num_hard_negatives=n)
  assert abs(float(loss) - rl) <= 1e-5 * abs(rl), (float(loss), rl)
  _close(qg.grad.cpu().numpy(), rdq, 1e-5, "dq")
  _close(cg.grad.cpu().numpy(), rdc, 1e-5, "dc")   # float atomics: order-dependent in the last bits only


def test_retrieval_task_hard_negatives_fused(ops, monkeypatch):
  import recommenders_b200 as tfrs
  B, C, d = 512, 1024, 64
  q = _rand((B, d), 61, 0.5); c = _rand((C, d), 62, 0.5)
  monkeypatch.setattr(ops, "scores", lambda *a, **k: (_ for _ in ()).throw(AssertionError("logits were materialised")))
  task = tfrs.tasks.Retrieval(num_hard_negatives=7, temperature=0.8)
  loss = task(q, c, compute_metrics=False)
  ref = orc.retrieval_loss(q.cpu().numpy(), c.cpu().numpy(), temperature=0.8, num_hard_negatives=7)
  assert abs(float(loss) - ref) <= 1e-5 * abs(ref), (float(loss), ref)


# ------------------------------------------------------------------------------------------------
# general tensor-core GEMM + low-rank Cross / MultiLayerDCN (dcn.py:131-148,178-186; multi_layer_dcn.py:136-153)
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("M,N,K,ta,tb", [(300, 200, 96, False, False), (1000, 130, 845, False, True), (257, 64, 5000, True, False),
                                         (129, 300, 3000, True, True), (4096, 845, 256, False, False)])
def test_gemm_tc_vs_float64(ops, M, N, K, ta, tb):
  a = _rand((K, M) if ta else (M, K), 71); b = _rand((N, K) if tb else (K, N), 72)
  out = ops.gemm_tc(a, b, ta, tb)
  a64 = a.cpu().numpy().astype(np.float64); b64 = b.cpu().numpy().astype(np.float64)
  ref = (a64.T if ta else a64) @ (b64.T if tb else b64)
  _close(out.cpu().numpy(), ref, 1e-5, "gemm_tc")   # split-fp16 products: ~2^-21 relative to |a||b|


def test_gemm_tc_transposed_operand_of_tiny_magnitude(ops):
  """max |a| ~ 1e-36 < 2^-113: the power-of-two rescale 2^exp is not a finite float on its own, yet the transposed
  operands (both read transposed here) must give finite images and the usual 1e-5 accuracy."""
  M, N, K = 257, 64, 5000
  a = _rand((K, M), 71, 1e-36); b = _rand((K, N), 72)
  out = ops.gemm_tc(a, b, True, False)
  ref = a.cpu().numpy().astype(np.float64).T @ b.cpu().numpy().astype(np.float64)
  _close(out.cpu().numpy(), ref, 1e-5, "gemm_tc")


def _lowrank_ref_grads(x0, x, U, V, b, g, diag):
  x0, x, U, V, g = (np.asarray(a, np.float64) for a in (x0, x, U, V, g))
  t = x @ U
  prod = t @ V + (0 if b is None else np.asarray(b, np.float64)) + diag * x
  gp = g * x0
  dt = gp @ V.T
  return {"out": x0 * prod + x, "dx0": g * prod, "dV": t.T @ gp, "dU": x.T @ dt, "dx": dt @ U.T + diag * gp + g, "db": gp.sum(0)}


@pytest.mark.parametrize("B,D,p,diag,bias", [(2048, 200, 64, 0.0, True), (1500, 130, 20, 0.5, True), (4096, 845, 256, 0.0, False)])
def test_cross_lowrank_tensor_cores_fwd_bwd(ops, B, D, p, diag, bias):
  x0 = _rand((B, D), 81, 0.5); x = _rand((B, D), 82, 0.5)
  U = _rand((D, p), 83, 0.05); V = _rand((p, D), 84, 0.05)
  b = _rand((D,), 85, 0.1) if bias else None
  g = _rand((B, D), 86)
  ts = [t.clone().requires_grad_(True) for t in (x0, x, U, V)]
  bg = None if b is None else b.clone().requires_grad_(True)
  out = ops.cross_lowrank(ts[0], ts[1], ts[2], ts[3], bg, diag)
  out.backward(g)
  ref = _lowrank_ref_grads(x0.cpu().numpy(), x.cpu().numpy(), U.cpu().numpy(), V.cpu().numpy(), None if b is None else b.cpu().numpy(),
                           g.cpu().numpy(), diag)
  # bar: 1e-5 relative to the tensor's scale (fp32 kernel vs float64 oracle, DESIGN section 2)
  _close(out.detach().cpu().numpy(), ref["out"], 1e-5, "out")
  _close(ts[0].grad.cpu().numpy(), ref["dx0"], 1e-5, "dx0")
  _close(ts[1].grad.cpu().numpy(), ref["dx"], 1e-5, "dx")
  _close(ts[2].grad.cpu().numpy(), ref["dU"], 1e-5, "dU")
  _close(ts[3].grad.cpu().numpy(), ref["dV"], 1e-5, "dV")
  if bg is not None:
    _close(bg.grad.cpu().numpy(), ref["db"], 1e-5, "dbias")


def test_cross_layer_and_multilayer_dcn_use_the_lowrank_tensor_core_path(ops, monkeypatch):
  import recommenders_b200 as tfrs
  B, D, p = 2048, 160, 32
  x0 = _rand((B, D), 91, 0.5)
  monkeypatch.setattr(ops, "matmul", lambda *a, **k: (_ for _ in ()).throw(AssertionError("unfused SGEMM path used")))
  layer = tfrs.layers.dcn.Cross(projection_dim=p, diag_scale=0.25)
  y = layer(x0)
  ref = orc.cross(x0.cpu().numpy(), None, None, layer.bias.detach().cpu().numpy(), 0.25,
                  U=layer.kernel_u.detach().cpu().numpy(), V=layer.kernel_v.detach().cpu().numpy())
  _close(y.detach().cpu().numpy(), ref, 1e-5, "Cross(projection_dim)")
  ml = tfrs.layers.feature_interaction.MultiLayerDCN(projection_dim=p, num_layers=3)
  y3 = ml(x0)
  ref3 = orc.multi_layer_dcn(x0.cpu().numpy(), [u.detach().cpu().numpy() for u in ml.u_kernels],
                             [v.detach().cpu().numpy() for v in ml.v_kernels], [b.detach().cpu().numpy() for b in ml.biases])
  _close(y3.detach().cpu().numpy(), ref3, 1e-5, "MultiLayerDCN")
  y3.sum().backward()
  assert all(u.grad is not None and torch.isfinite(u.grad).all() for u in ml.u_kernels)


# ------------------------------------------------------------------------------------------------
# gather: hot rows staged in shared memory (skewed ids)
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("idt", [torch.int32, torch.int64])
@pytest.mark.parametrize("dim", [32, 64])
def test_gather_hot_rows_bit_exact(ops, idt, dim):
  g = torch.Generator(device="cuda"); g.manual_seed(101)
  tables = [torch.randn((5000, dim), generator=g, device="cuda") for _ in range(3)]
  n = 4099
  u = torch.rand((3, n), generator=g, device="cuda", dtype=torch.float64)
  ids = [((u[t] ** 6) * 5000).to(idt) for t in range(3)]          # heavily skewed towards row 0 (hot rows = low ids)
  ids[1][::3] = 4999; ids[2][:64] = -1                             # cold rows and out-of-range ids in the same chunk
  out = ops.gather(tables, ids)
  exp = np.concatenate([orc.gather(t.cpu().numpy(), i.cpu().numpy()) for t, i in zip(tables, ids)], 1)
  assert np.array_equal(out.cpu().numpy(), exp)


# ------------------------------------------------------------------------------------------------
# multi-head queries: maxsim folded into the blocked loss (tasks/retrieval.py:172-176)
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B,H,C,d,temp,weighted", [(2, 2, 3, 3, None, False), (300, 4, 500, 32, 0.5, True), (1000, 2, 1000, 64, None, False)])
def test_maxsim_loss_fused(ops, B, H, C, d, temp, weighted):
  q = _rand((B, H, d), 111, 0.5); c = _rand((C, d), 112, 0.5)
  w = (torch.rand((B,), device="cuda") + 0.5) if weighted else None
  qg = q.clone().requires_grad_(True); cg = c.clone().requires_grad_(True)
  loss = ops.inbatch_softmax_maxsim_loss(qg, cg, w, temp)
  loss.backward()
  ref = orc.retrieval_loss(q.cpu().numpy(), c.cpu().numpy(), None if w is None else w.cpu().numpy(), temperature=temp)
  assert abs(float(loss) - ref) <= 1e-5 * abs(ref), (float(loss), ref)
  # float64 gradient: G goes to the arg-max head
  q64 = q.cpu().numpy().astype(np.float64); c64 = c.cpu().numpy().astype(np.float64)
  t = 1.0 if temp is None else temp
  sh = np.einsum("bhd,cd->bhc", q64, c64)
  s = sh.max(1) / t
  m = s.max(1, keepdims=True); p = np.exp(s - m); p /= p.sum(1, keepdims=True)
  g = (p - np.eye(B, C)) * ((np.ones(B) if w is None else w.cpu().numpy().astype(np.float64))[:, None] / t)
  sel = (sh == sh.max(1, keepdims=True)).astype(np.float64)
  sel /= sel.sum(1, keepdims=True)
  gh = sel * g[:, None, :]
  _close(qg.grad.cpu().numpy(), np.einsum("bhc,cd->bhd", gh, c64), 1e-5, "dq")
  _close(cg.grad.cpu().numpy(), np.einsum("bhc,bhd->cd", gh, q64), 1e-5, "dc")


def test_retrieval_task_maxsim_known_answer(ops, monkeypatch):
  """retrieval_test.py:255-298: q [2,2,3] -> maxsim scores [[2,5,5],[3,7,7]]; the task must not build them with eager ops."""
  import recommenders_b200 as tfrs
  q = torch.tensor([[[0., 1, 0], [1, 1, 0]], [[0, 1, 1], [1, 0, 1]]], device="cuda")   # any heads: compare with the oracle
  c = torch.tensor([[0., 1, 0], [0, 1, 1], [1, 1, 0]], device="cuda")
  monkeypatch.setattr(ops, "scores", lambda *a, **k: (_ for _ in ()).throw(AssertionError("logits were materialised")))
  loss = tfrs.tasks.Retrieval()(q, c, compute_metrics=False)
  ref = orc.retrieval_loss(q.cpu().numpy(), c.cpu().numpy())
  assert abs(float(loss) - ref) <= 1e-6 * max(1.0, abs(ref))


def test_cross_stack_reuses_the_epilogue_statistic(ops):
  """x = cross(x0, x) chains: layer l+1 takes max|x| from layer l's epilogue instead of a pass over x -- identical bits."""
  import recommenders_b200 as tfrs
  B, D = 2304, 200
  x0 = _rand((B, D), 121, 0.5)
  layers = [tfrs.layers.dcn.Cross() for _ in range(3)]
  with torch.no_grad():
    x = x0
    for l in layers:
      x = l(x0, x)
      am, ver, ptr_ = x._tfrs_amax
      assert ver == x._version and ptr_ == x.data_ptr()
      assert int(am.item()) == int(x.abs().max().view(torch.int32).item())      # float bits of max |out|
    y = x0
    for l in layers:
      y = l(x0, y.clone())                                                        # a copy carries no statistic: full pass
  assert torch.equal(x, y)
  ref = orc.cross(x0.cpu().numpy(), None, layers[0].kernel.detach().cpu().numpy(), layers[0].bias.detach().cpu().numpy())
  _close(layers[0](x0).detach().cpu().numpy(), ref, 1e-5, "first layer")
  # an in-place edit invalidates the statistic (version check): the result must still be right
  with torch.no_grad():
    z = layers[0](x0)
    z.mul_(64.0)
    out = layers[1](x0, z)
    assert torch.equal(out, layers[1](x0, z.clone()))
  # gradients still flow through the stack
  xs = x0.clone().requires_grad_(True)
  h = xs
  for l in layers:
    h = l(xs, h)
  h.sum().backward()
  assert torch.isfinite(xs.grad).all() and all(torch.isfinite(l.kernel.grad).all() for l in layers)
