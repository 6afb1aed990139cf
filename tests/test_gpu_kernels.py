"""GPU parity tests (run with -m gpu on an H100): every kernel of libtfrs_b200.so, called through the C ABI
(via recommenders_b200.ops), against the CPU oracle on the same seeded inputs.
Bar: bit-exact for scores / indices / gathered rows / Adagrad state; 1e-5 relative for the fp32
softmax loss, its gradients and the Cross layer (tolerance stated per test)."""
import numpy as np
import pytest
import torch

from oracle import oracle as orc

pytestmark = pytest.mark.gpu


def dev():
  return torch.device("cuda", 0)


def cu(a):
  return torch.from_numpy(np.ascontiguousarray(a)).to(dev())


@pytest.fixture(scope="module")
def ops():
  from recommenders_b200 import ops as o
  return o


@pytest.mark.parametrize("Q,N,d,k", [(3, 128, 4, 5), (16, 1024, 4, 10), (7, 1000, 64, 100), (33, 5000, 33, 17),
                                     (130, 3001, 128, 100), (1, 1, 8, 1), (5, 50, 16, 100), (64, 20000, 64, 100)])
def test_topk_scan_bit_exact(ops, Q, N, d, k):
  rng = np.random.RandomState(Q * 1000 + N)
  q = rng.normal(size=(Q, d)).astype(np.float32); c = rng.normal(size=(N, d)).astype(np.float32)
  es, ei = orc.topk_scan(q, c, k)
  s, i = ops.topk_scan(cu(q), cu(c), k)
  assert s.shape == es.shape
  np.testing.assert_array_equal(i.cpu().numpy(), ei)
  np.testing.assert_array_equal(s.cpu().numpy().view(np.uint32), es.view(np.uint32))


def test_topk_scan_ties_and_offsets(ops):
  q = np.ones((2, 4), np.float32); c = np.ones((300, 4), np.float32)
  s, i = ops.topk_scan(cu(q), cu(c), 7, index_offset=1000)
  np.testing.assert_array_equal(i.cpu().numpy(), np.tile(np.arange(1000, 1007), (2, 1)))
  # duplicate rows scattered over the corpus: lowest index wins
  rng = np.random.RandomState(1)
  base = rng.normal(size=(50, 8)).astype(np.float32)
  c2 = np.concatenate([base, base, base], 0); q2 = rng.normal(size=(9, 8)).astype(np.float32)
  es, ei = orc.topk_scan(q2, c2, 20)
  s, i = ops.topk_scan(cu(q2), cu(c2), 20)
  np.testing.assert_array_equal(i.cpu().numpy(), ei)


def test_topk_scan_streaming_state(ops):
  rng = np.random.RandomState(7)
  q = rng.normal(size=(11, 16)).astype(np.float32); c = rng.normal(size=(700, 16)).astype(np.float32)
  es, ei = orc.topk_scan(q, c, 25)
  state = (torch.zeros((11, 0), device=dev()), torch.zeros((11, 0), dtype=torch.int64, device=dev()))
  off = 0
  for chunk in (3, 100, 17, 580):  # ragged chunks, first ones smaller than k
    state = ops.topk_scan(cu(q), cu(c[off:off + chunk]), 25, index_offset=off, state=state)
    off += chunk
  np.testing.assert_array_equal(state[1].cpu().numpy(), ei)
  np.testing.assert_array_equal(state[0].cpu().numpy(), es)


def test_topk_scan_multichunk_workspace(ops):
  # Q large enough that the score chunk is cut (nc < N) -> exercises the internal chunk loop + carried state
  rng = np.random.RandomState(3)
  Q, N, d, k = 9000, 9000, 8, 10
  q = rng.normal(size=(Q, d)).astype(np.float32); c = rng.normal(size=(N, d)).astype(np.float32)
  s, i = ops.topk_scan(cu(q), cu(c), k)
  es, ei = orc.topk_scan(q[:200], c, k)
  np.testing.assert_array_equal(i[:200].cpu().numpy(), ei)
  np.testing.assert_array_equal(s[:200].cpu().numpy(), es)


def test_topk_merge(ops):
  rng = np.random.RandomState(5)
  q = rng.normal(size=(13, 8)).astype(np.float32); c = rng.normal(size=(900, 8)).astype(np.float32)
  full_s, full_i = orc.topk_scan(q, c, 50)
  parts = [ops.topk_scan(cu(q), cu(c[o:o + 300]), 50, index_offset=o) for o in (0, 300, 600)]
  ms, mi = ops.topk_merge(torch.stack([p[0] for p in parts]), torch.stack([p[1] for p in parts]), 50)
  np.testing.assert_array_equal(mi.cpu().numpy(), full_i)
  np.testing.assert_array_equal(ms.cpu().numpy(), full_s)


def test_scores_and_rowdot_bit_exact(ops):
  rng = np.random.RandomState(11)
  q = rng.normal(size=(70, 37)).astype(np.float32); c = rng.normal(size=(301, 37)).astype(np.float32)
  np.testing.assert_array_equal(ops.scores(cu(q), cu(c)).cpu().numpy(), orc.scores(q, c))
  rd = ops.rowwise_dot(cu(q), cu(c[:70])).cpu().numpy()
  np.testing.assert_array_equal(rd, np.diag(orc.scores(q, c[:70])))


@pytest.mark.parametrize("idt", [np.int32, np.int64])
def test_gather_bit_exact(ops, idt):
  rng = np.random.RandomState(2)
  tabs = [rng.normal(size=(r, d)).astype(np.float32) for r, d in ((1000, 64), (50, 32), (7, 8), (300, 5))]
  n = 777
  ids = [rng.randint(0, t.shape[0], size=n).astype(idt) for t in tabs]
  ids[1][5] = -1; ids[1][6] = 50  # out of range -> zero rows
  exp = np.concatenate([orc.gather(t, i) for t, i in zip(tabs, ids)], 1)
  out = ops.gather([cu(t) for t in tabs], [cu(i) for i in ids])
  np.testing.assert_array_equal(out.cpu().numpy(), exp)
  # vectorised path (all dims % 4 == 0) with a padded leading dimension
  out2 = torch.zeros((n, 104), device=dev())
  ops.gather([cu(tabs[0]), cu(tabs[1])], [cu(ids[0]), cu(ids[1])], out=out2)
  np.testing.assert_array_equal(out2[:, :96].cpu().numpy(), exp[:, :96])
  assert float(out2[:, 96:].abs().sum()) == 0.0


@pytest.mark.parametrize("inside", [True, False])
@pytest.mark.parametrize("n,rows", [(64, 10), (5000, 300), (20000, 100000)])
def test_sparse_adagrad_bit_exact(ops, inside, n, rows):
  rng = np.random.RandomState(n)
  d = 64
  table = rng.uniform(-0.05, 0.05, size=(rows, d)).astype(np.float32)
  accum = np.full((rows, d), 0.1, np.float32)
  ids = (rng.zipf(1.3, size=n) % rows).astype(np.int64)  # hot rows + many duplicates
  g = rng.normal(size=(n, d)).astype(np.float32)
  et, ea = orc.sparse_adagrad(table, accum, ids, g, lr=0.5, eps=1e-7, eps_inside_sqrt=inside)
  t, a = cu(table), cu(accum)
  ops.sparse_adagrad_(t, a, cu(ids), cu(g), 0.5, 1e-7, inside)
  np.testing.assert_array_equal(a.cpu().numpy(), ea)
  np.testing.assert_array_equal(t.cpu().numpy(), et)


@pytest.mark.parametrize("B,C,d,temp,weighted", [(2, 2, 3, None, False), (64, 64, 16, None, True), (300, 517, 64, 0.5, True),
                                                 (1024, 1024, 64, None, False)])
def test_inbatch_softmax_loss_and_grads(ops, B, C, d, temp, weighted):
  """fp32 kernel vs float64 oracle: 1e-5 relative on the loss, 1e-5 of the gradient scale on dq/dc."""
  rng = np.random.RandomState(B + C)
  q = rng.normal(size=(B, d)).astype(np.float32) * 0.5; c = rng.normal(size=(C, d)).astype(np.float32) * 0.5
  w = rng.uniform(size=(B,)).astype(np.float32) if weighted else None
  exp = orc.retrieval_loss(q, c, sample_weight=w, temperature=temp)
  edq, edc = orc.retrieval_loss_grads(q, c, sample_weight=w, temperature=temp)
  tq = cu(q).requires_grad_(True); tc = cu(c).requires_grad_(True)
  loss = ops.inbatch_softmax_loss(tq, tc, None if w is None else cu(w), temp)
  loss.backward()
  assert abs(float(loss) - exp) <= 1e-5 * abs(exp)
  for got, ref in ((tq.grad, edq), (tc.grad, edc)):
    err = np.abs(got.cpu().numpy().astype(np.float64) - ref).max()
    assert err <= 1e-5 * np.abs(ref).max()


@pytest.mark.parametrize("B,D,diag,bias", [(1, 3, 0.0, False), (257, 845, 0.0, True), (100, 64, 1.0, True), (5000, 130, 0.5, False),
                                           (4096, 845, 0.0, True), (1500, 64, 0.25, False), (2048, 200, 0.0, True),
                                           (2048, 1100, 0.25, True)])   # D > 1024: one accumulation chain over all of K
def test_cross_fwd_bwd(ops, B, D, diag, bias):
  """1e-5 relative to the output scale (fp32 kernel vs float64 oracle)."""
  rng = np.random.RandomState(B + D)
  x0 = rng.uniform(size=(B, D)).astype(np.float32); x = rng.uniform(size=(B, D)).astype(np.float32)
  W = (rng.normal(size=(D, D)) * 0.05).astype(np.float32)
  b = rng.normal(size=(D,)).astype(np.float32) if bias else None
  g = rng.normal(size=(B, D)).astype(np.float32)
  exp = orc.cross(x0, x, W, b, diag)
  edx0, edx, edW, edb = orc.cross_grads(x0, x, W, b, g, diag)
  t = [cu(a).requires_grad_(True) for a in (x0, x, W)]
  tb = cu(b).requires_grad_(True) if bias else None
  out = ops.cross(t[0], t[1], t[2], tb, diag)
  np.testing.assert_allclose(out.detach().cpu().numpy(), exp, rtol=1e-5, atol=1e-5 * np.abs(exp).max())
  out.backward(cu(g))
  for got, ref in ((t[0].grad, edx0), (t[1].grad, edx), (t[2].grad, edW)) + (((tb.grad, edb),) if bias else ()):
    err = np.abs(got.cpu().numpy().astype(np.float64) - ref).max()
    assert err <= 1e-5 * np.abs(ref).max(), err


def test_errors_cross_the_abi(ops):
  with pytest.raises(ValueError):
    ops.topk_scan(cu(np.zeros((2, 4), np.float32)), cu(np.zeros((8, 4), np.float32)), 5000)
  with pytest.raises(RuntimeError):
    ops.topk_scan(torch.zeros((2, 4)), torch.zeros((8, 4)), 3)  # CPU tensors: no fallback


def test_cross_tensor_core_matches_cuda_core(ops):
  """The wgmma Cross forward (fp16 hi/lo split) against the exact CUDA-core kernel: 1e-5 of the output scale."""
  rng = np.random.RandomState(0)
  B, D = 8192, 845
  x0 = cu(rng.uniform(size=(B, D)).astype(np.float32)); x = cu(rng.normal(size=(B, D)).astype(np.float32))
  W = cu((rng.normal(size=(D, D)) * 0.05).astype(np.float32)); b = cu(rng.normal(size=(D,)).astype(np.float32))
  tc = ops.cross(x0, x, W, b, 0.5)
  old = ops.CROSS_TC_MIN_B
  try:
    ops.CROSS_TC_MIN_B = 1 << 60
    ref = ops.cross(x0, x, W, b, 0.5)
  finally:
    ops.CROSS_TC_MIN_B = old
  err = float((tc - ref).abs().max()); scale = float(ref.abs().max())
  assert err <= 1e-5 * scale, (err, scale)
  # weights updated in place -> the cached image must be rebuilt
  W.mul_(2.0)
  tc2 = ops.cross(x0, x, W, b, 0.5)
  ops.CROSS_TC_MIN_B = 1 << 60
  try:
    ref2 = ops.cross(x0, x, W, b, 0.5)
  finally:
    ops.CROSS_TC_MIN_B = old
  assert float((tc2 - ref2).abs().max()) <= 1e-5 * float(ref2.abs().max())


@pytest.mark.parametrize("idt", [np.int32, np.int64])
def test_gather_uniform_tables_fast_path(ops, idt):
  """All tables the same width (the DCN-v2 / two-tower shape): table-fastest kernel, concatenated output with padding."""
  rng = np.random.RandomState(9)
  T, V, D, n = 5, 3000, 32, 1234
  tabs = [rng.normal(size=(V, D)).astype(np.float32) for _ in range(T)]
  ids = [rng.randint(0, V, size=n).astype(idt) for _ in range(T)]
  ids[2][7] = V; ids[4][0] = -3   # out of range -> zero rows
  exp = np.concatenate([orc.gather(t, i) for t, i in zip(tabs, ids)], 1)
  out = torch.full((n, T * D + 8), -7.0, device=dev())
  ops.gather([cu(t) for t in tabs], [cu(i) for i in ids], out=out)
  np.testing.assert_array_equal(out[:, :T * D].cpu().numpy(), exp)
  assert float((out[:, T * D:] + 7.0).abs().sum()) == 0.0   # padding columns untouched


@pytest.mark.parametrize("B,C,d,temp,weighted,scale", [(2, 2, 3, None, False, 0.5), (300, 517, 64, 0.5, True, 0.5),
                                                       (1024, 1024, 64, None, False, 0.5), (700, 9000, 100, 0.05, True, 0.1),
                                                       (2500, 2500, 32, None, True, 1.0)])
def test_inbatch_softmax_tensor_core_forward(ops, B, C, d, temp, weighted, scale):
  """wgmma forward (hi/lo fp16 split, online log-sum-exp epilogue) vs the float64 oracle: 1e-5 relative on the
  loss, 1e-5 absolute-or-relative on every row's logsumexp; and it must agree with the exact CUDA-core forward."""
  rng = np.random.RandomState(B + C + d)
  q = rng.normal(size=(B, d)).astype(np.float32) * scale; c = rng.normal(size=(C, d)).astype(np.float32) * scale
  w = rng.uniform(size=(B,)).astype(np.float32) if weighted else None
  inv_t = 1.0 if temp is None else 1.0 / temp
  exp = orc.retrieval_loss(q, c, sample_weight=w, temperature=temp)
  s = (q.astype(np.float64) @ c.astype(np.float64).T) * inv_t
  m = s.max(1)
  elses = m + np.log(np.exp(s - m[:, None]).sum(1))
  loss, lse = ops.inbatch_softmax_tc(cu(q), cu(c), None if w is None else cu(w), inv_t)
  assert abs(float(loss) - exp) <= 1e-5 * abs(exp)
  np.testing.assert_allclose(lse.cpu().numpy().astype(np.float64), elses, rtol=1e-5, atol=1e-5)
  if B >= ops.SOFTMAX_TC_MIN_B:  # the autograd op takes this path: gradients (exact kernels, tensor-core lse) stay in tolerance
    edq, edc = orc.retrieval_loss_grads(q, c, sample_weight=w, temperature=temp)
    tq = cu(q).requires_grad_(True); tc = cu(c).requires_grad_(True)
    l2 = ops.inbatch_softmax_loss(tq, tc, None if w is None else cu(w), temp)
    l2.backward()
    assert float(l2) == float(loss)
    for got, ref in ((tq.grad, edq), (tc.grad, edc)):
      err = np.abs(got.cpu().numpy().astype(np.float64) - ref).max()
      assert err <= 1e-5 * np.abs(ref).max()


@pytest.mark.parametrize("B,C,d,temp,weighted,scale", [(2, 2, 3, None, False, 0.5), (128, 128, 64, None, False, 0.5),
                                                       (300, 517, 64, 0.5, True, 0.5), (1024, 1024, 64, None, False, 0.5),
                                                       (700, 5000, 40, 0.05, True, 0.1), (2500, 2500, 32, None, True, 1.5),
                                                       (1300, 1300, 64, 0.1, True, 0.3)])
def test_inbatch_softmax_tensor_core_backward(ops, B, C, d, temp, weighted, scale):
  """wgmma backward (S = X.Y^T in registers, dX += G.Y with G as the register A operand) vs the float64 oracle:
  1e-5 of the gradient scale on dq and dc, with lse from the tensor-core forward and a non-unit upstream gradient."""
  rng = np.random.RandomState(B + C + d + 1)
  q = rng.normal(size=(B, d)).astype(np.float32) * scale; c = rng.normal(size=(C, d)).astype(np.float32) * scale
  w = rng.uniform(size=(B,)).astype(np.float32) if weighted else None
  if w is not None:
    w[0] = 0.0  # a masked example
  inv_t = 1.0 if temp is None else 1.0 / temp
  gl = 0.37
  edq, edc = orc.retrieval_loss_grads(q, c, sample_weight=w, temperature=temp)
  _, lse = ops.inbatch_softmax_tc(cu(q), cu(c), None if w is None else cu(w), inv_t)
  dq, dc = ops.inbatch_softmax_tc_bwd(cu(q), cu(c), lse, None if w is None else cu(w), inv_t, torch.tensor([gl], device="cuda"))
  for got, ref in ((dq, edq * gl), (dc, edc * gl)):
    err = np.abs(got.cpu().numpy().astype(np.float64) - ref).max()
    assert err <= 1e-5 * np.abs(ref).max(), (err, np.abs(ref).max())


def test_inbatch_softmax_tensor_core_backward_full_size(ops):
  """cfg3 size (B = C = 16384, d = 64): the tensor-core backward against the exact CUDA-core backward with the same
  lse -- a consistency check between two fp32 paths, each with its own accumulation error, hence 2e-5 of the
  gradient scale here; the parity bar proper (1e-5 against float64) is
  tests/test_gpu_round2.py::test_cfg3_full_size_loss_and_gradients_vs_float64."""
  g = torch.Generator(device="cuda"); g.manual_seed(11)
  B, d = 16384, 64
  q = (torch.rand((B, d), generator=g, device="cuda") - 0.5) * 0.6
  c = (torch.rand((B, d), generator=g, device="cuda") - 0.5) * 0.6
  w = torch.rand((B,), generator=g, device="cuda")
  _, lse = ops.inbatch_softmax_tc(q, c, w, 2.0)
  tq, tc = ops.inbatch_softmax_tc_bwd(q, c, lse, w, 2.0)
  eq, ec = ops.inbatch_softmax_bwd_exact(q, c, lse, w, 2.0)
  for a, b in ((tq, eq), (tc, ec)):
    assert float((a - b).abs().max()) <= 2e-5 * float(b.abs().max())


@pytest.mark.parametrize("B,C,d,temp,weighted", [(600, 600, 64, 0.2, True), (1024, 3000, 32, None, False), (2500, 2500, 48, 0.5, True)])
def test_inbatch_softmax_with_sampling_probability_correction(ops, B, C, d, temp, weighted):
  """Fused tensor-core loss with the per-candidate bias -log(clip(p, 1e-6, 1)) (retrieval.py:190-192): loss vs the
  oracle's materialised path, gradients vs float64, and the Retrieval task routes the option to the fused kernels."""
  import recommenders_b200 as tfrs
  rng = np.random.RandomState(B + C + d + 7)
  q = rng.normal(size=(B, d)).astype(np.float32) * 0.4; c = rng.normal(size=(C, d)).astype(np.float32) * 0.4
  w = rng.uniform(size=(B,)).astype(np.float32) if weighted else None
  prob = rng.uniform(1e-7, 1.0, size=(C,)).astype(np.float32)   # includes values below the 1e-6 clip
  exp = orc.retrieval_loss(q, c, sample_weight=w, temperature=temp, candidate_sampling_probability=prob)
  t = 1.0 if temp is None else temp
  bias = -np.log(np.clip(prob.astype(np.float64), 1e-6, 1.0))
  s = q.astype(np.float64) @ c.astype(np.float64).T / t + bias[None, :]
  p = np.exp(s - s.max(1, keepdims=True)); p /= p.sum(1, keepdims=True)
  g = (p - np.eye(B, C)) * (np.ones(B) if w is None else w.astype(np.float64))[:, None] / t
  edq, edc = g @ c.astype(np.float64), g.T @ q.astype(np.float64)
  assert ops.inbatch_softmax_bias_supported(B, C, d)
  tq = cu(q).requires_grad_(True); tc = cu(c).requires_grad_(True)
  task = tfrs.tasks.Retrieval(temperature=temp)
  loss = task(tq, tc, sample_weight=None if w is None else cu(w), candidate_sampling_probability=cu(prob), compute_metrics=False)
  loss.backward()
  assert abs(float(loss) - exp) <= 1e-5 * abs(exp)
  for got, ref in ((tq.grad, edq), (tc.grad, edc)):
    err = np.abs(got.cpu().numpy().astype(np.float64) - ref).max()
    assert err <= 1e-5 * np.abs(ref).max()
  # the fused op itself, and the materialised path of the task on the same data (forced by a tiny batch-metric-free slice)
  direct = ops.inbatch_softmax_loss(cu(q), cu(c), None if w is None else cu(w), temp, cu(bias.astype(np.float32)))
  assert abs(float(direct) - exp) <= 1e-5 * abs(exp)
