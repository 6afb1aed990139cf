"""Edge cases of the two exact CUDA-core kernels every tensor-core path is checked against: the SGEMM (csrc/sgemm.cuh) and
the per-query row select (csrc/rowselect.cuh), through the exact top-K scan and list merges (csrc/topk.cu), the exact
Dense and Cross layers (csrc/dense.cu, csrc/cross.cu) and the MovieLens dense route (csrc/eval_topk.cu); and the
tensor-core top-K (csrc/topk_tc.cu) on a corpus that does not start on a 16-byte boundary.

The reference of every product is the C oracle's sequential fmaf chain from +0.0f (oracle.scores).  Transposition only
changes the memory layout, so one reference serves all four SGEMM modes.  Everything is compared bit for bit
(view(np.uint32)) unless a test states a bar.  The case lists below are module constants: tests/test_exact_anchor_cases.py
reads the kernels' constants back from the sources and checks on a CPU that these lists still hit every edge.
"""
import numpy as np
import pytest
import torch

from oracle import oracle as orc

pytestmark = pytest.mark.gpu

# ---- csrc/sgemm.cuh: SG_BM = SG_BN = 128, SG_BK = 16, the 64-column skinny tile for N <= 64
SG_MODES = [(False, False), (False, True), (True, False), (True, True)]
SG_M = [1, 127, 128, 129, 257]              # one row; both sides of one 128-row tile; a third, one-row tile
SG_N = [1, 63, 64, 65, 127, 128, 129]       # skinny tile up to 64, 128-column tiles above; both sides of each tile
SG_K = [0, 1, 2, 3, 4, 5, 15, 16, 17, 18, 31, 33, 100]   # every K % 4 tail of the float4 loaders below and above one
#                                                       16-slab; < / = / > one slab, two slabs +-1, six and a tail
# (M, N, K): K walks its list while M and N cycle through theirs, so every M, N and K value is run in every mode
SG_CASES = [(SG_M[i % len(SG_M)], SG_N[i % len(SG_N)], K) for i, K in enumerate(SG_K)] + \
           [(SG_M[(i + 2) % len(SG_M)], SG_N[(i + 4) % len(SG_N)], K) for i, K in enumerate(SG_K)]
SG_OFFSETS = [1, 2, 3]                      # base 4, 8 and 12 bytes into the storage: the scalar loader fallback
SG_LD_PAD = [1, 4]                          # ld = width + 1 (fallback), width + 4 (float4 loads with a row gap)
SG_LD_SHAPES = [(129, 65, 36), (70, 130, 17)]   # K % 4 == 0 (so ld = K + 4 keeps the float4 path) and a K % 16 == 1 tail
SG_NEG_ZERO_K = [1, 3, 5, 17, 33, 100]      # not multiples of SG_BK: the partial-slab loop carries the chain's last term

# ---- split-K over the batch (sgemm_batch_splits: ranges of about 4096 rows, at most 16) and DENSE_COL_SPLITS = 64
SPLIT_B = [4096, 4097, 8193, 65536, 65537, 70000]   # 1 range / 2 / 3 / 16 / the cap (17 wanted) / the cap, ragged
DENSE_BWD_KN = (20, 40)     # K < 64: the exact backward at any batch size
CROSS_BWD_D = 24            # D < 64: the exact Cross at any batch size
DENSE_FWD_CASES = [(257, 33, 16), (257, 33, 17),    # DENSE_NARROW_N = 16: the warp-per-row kernel, then the SGEMM
                   (129, 100, 64), (127, 5, 65), (1, 17, 129), (300, 31, 128), (2000, 40, 63)]
SIGMOID_ULP = 4             # expf (<= 2 ulp), 1 + e and the IEEE division

# ---- csrc/rowselect.cuh: cap = max(1024, pow2_ceil(2k)), compaction when the free room drops below cap / 4
SEL_K = [1, 2, 511, 512, 513, 1023, 1024, 1025, 2047, 2048]
SEL_PATTERNS = ["random", "ascending", "equal", "inf", "zeros"]
SEL_MANY = 5                # N = SEL_MANY * cap + 17: several compactions
# chunk loop of the exact scan (scan_plan: 256 MB of scores per chunk, >= 1024 columns, multiples of 128)
CHUNK_QNK = (40000, 3 * 1664 + 77, 600)
# workspace-shrink branch: (Q, N, k, extra bytes above 2 * state_bytes)
SHRINK_CASES = [(64, 10000, 100, 64 * 4096 + 512), (64, 10000, 100, 64 * 8192 + 1000), (3, 7000, 2048, 3 * 4096 + 256)]
# sorting merge: (n_lists, k_in, k_out), n_lists * k_in > cap(k_out)
SORT_MERGE_CASES = [(3, 1500, 2048), (5, 1000, 1025), (9, 600, 2047), (2, 700, 512)]
# sorted-list (tree) merge: n_lists around MS_MAX_LISTS = 64, region * 24 around 160 KB
TREE_MERGE_CASES = [(64, 16, 100), (65, 16, 100), (2, 3413, 2048), (2, 3414, 2048), (4, 1706, 1500), (4, 1707, 1500)]
OVERRIDE_K = 1025

# ---- the tensor-core top-K on an unaligned corpus
TC_UNALIGNED_D = [32, 36, 64]   # exact_score's d % 32 == 0 loop, its d % 4 == 0 loop, the d == 64 band loader
TC_UNALIGNED_OFF = [1, 2, 3]    # corpus 4, 8 and 12 bytes into its storage
TC_QNK = (64, 20000, 50)


@pytest.fixture(scope="module")
def ops():
  from recommenders_b200 import ops as o
  return o


def dev():
  return torch.device("cuda", 0)


def cu(a):
  return torch.from_numpy(np.ascontiguousarray(a)).to(dev())


def bits(a):
  a = a.detach().cpu().numpy() if isinstance(a, torch.Tensor) else np.asarray(a)
  return np.ascontiguousarray(a, np.float32).view(np.uint32)


def assert_bits(got, exp, msg=""):
  np.testing.assert_array_equal(bits(got), bits(exp), err_msg=msg)


def cdiv(a, b):
  return -(-a // b)


# ================================================================================================
# SGEMM
# ================================================================================================
def _stored(op, trans):
  """The array a kernel reads for the logical operand `op`: op itself, or its transpose laid out row-major."""
  return np.ascontiguousarray(op.T if trans else op)


def _operands(M, N, K, seed):
  rng = np.random.RandomState(seed)
  return rng.normal(size=(M, K)).astype(np.float32), rng.normal(size=(K, N)).astype(np.float32)


def _ref(opA, opB):
  return orc.scores(opA, opB.T)   # C[m, n] = chain over k of opA[m, k] * opB[k, n]


def _raw_sgemm(ops, ta, tb, M, N, K, a, lda, b, ldb, c, ldc, accumulate=False):
  from recommenders_b200._ffi import ptr, stream
  return ops.lib().tfrs_sgemm_f32(int(ta), int(tb), M, N, K, ptr(a), lda, ptr(b), ldb, ptr(c), ldc, int(accumulate), stream())


@pytest.mark.parametrize("ta,tb", SG_MODES)
@pytest.mark.parametrize("M,N,K", SG_CASES)
def test_sgemm_tile_and_slab_edges(ops, ta, tb, M, N, K):
  opA, opB = _operands(M, N, K, M * 1000 + N * 10 + K)
  got = ops.sgemm(cu(_stored(opA, ta)), cu(_stored(opB, tb)), ta, tb)   # K = 0: empty operands, NULL data pointers
  assert tuple(got.shape) == (M, N)
  assert_bits(got, _ref(opA, opB))


@pytest.mark.parametrize("ta,tb", SG_MODES)
@pytest.mark.parametrize("off", SG_OFFSETS)
def test_sgemm_unaligned_bases(ops, ta, tb, off):
  """A and B views that start 4, 8 or 12 bytes into their storage: the float4 loaders fall back to scalar loads."""
  for M, N, K in SG_LD_SHAPES:
    opA, opB = _operands(M, N, K, 7 * off + M)
    sa, sb = _stored(opA, ta), _stored(opB, tb)
    store_a = torch.zeros(off + sa.size + 3, device=dev()); store_b = torch.zeros(off + sb.size + 3, device=dev())
    a = store_a[off:off + sa.size].view(sa.shape); a.copy_(cu(sa))
    b = store_b[off:off + sb.size].view(sb.shape); b.copy_(cu(sb))
    assert a.data_ptr() % 16 == 4 * off and b.data_ptr() % 16 == 4 * off
    aligned = ops.sgemm(cu(sa), cu(sb), ta, tb)
    got = ops.sgemm(a, b, ta, tb)
    assert_bits(got, aligned)
    assert_bits(got, _ref(opA, opB))


@pytest.mark.parametrize("ta,tb", SG_MODES)
@pytest.mark.parametrize("pad", SG_LD_PAD)
def test_sgemm_padded_leading_dims(ops, ta, tb, pad):
  """lda / ldb = row width + 1 (float4 off) and + 4 (float4 on, rows with a gap), through the C ABI."""
  for M, N, K in SG_LD_SHAPES:
    opA, opB = _operands(M, N, K, 11 * pad + N)
    sa, sb = _stored(opA, ta), _stored(opB, tb)
    lda, ldb = sa.shape[1] + pad, sb.shape[1] + pad
    a = torch.full((sa.shape[0], lda), float("nan"), device=dev()); a[:, :sa.shape[1]] = cu(sa)
    b = torch.full((sb.shape[0], ldb), float("nan"), device=dev()); b[:, :sb.shape[1]] = cu(sb)
    c = torch.empty((M, N), device=dev())
    assert _raw_sgemm(ops, ta, tb, M, N, K, a, lda, b, ldb, c, N) == 0
    assert_bits(c, ops.sgemm(cu(sa), cu(sb), ta, tb))
    assert_bits(c, _ref(opA, opB))


@pytest.mark.parametrize("ta,tb", SG_MODES)
def test_sgemm_strided_output_and_accumulate(ops, ta, tb):
  """ldc > N through a column slice of a wider buffer: the columns outside keep their sentinel; accumulate adds the
  product to the output with one IEEE add."""
  sentinel = -1234.5
  for M, N, K in [(129, 65, 17), (1, 129, 33), (257, 64, 100)]:
    opA, opB = _operands(M, N, K, M + N + K)
    S = _ref(opA, opB)
    buf = torch.full((M, N + 7), sentinel, device=dev())
    out = buf[:, 3:3 + N]
    ops.sgemm(cu(_stored(opA, ta)), cu(_stored(opB, tb)), ta, tb, out=out)
    h = buf.cpu().numpy()
    assert_bits(h[:, 3:3 + N], S)
    assert (h[:, :3] == sentinel).all() and (h[:, 3 + N:] == sentinel).all()
    C0 = np.random.RandomState(K).normal(size=(M, N)).astype(np.float32)
    out.copy_(cu(C0))
    ops.sgemm(cu(_stored(opA, ta)), cu(_stored(opB, tb)), ta, tb, out=out, accumulate=True)
    h = buf.cpu().numpy()
    assert_bits(h[:, 3:3 + N], C0 + S)     # float32 + float32: one rounding
    assert (h[:, :3] == sentinel).all() and (h[:, 3 + N:] == sentinel).all()


@pytest.mark.parametrize("ta,tb", SG_MODES)
@pytest.mark.parametrize("K", SG_NEG_ZERO_K)
def test_sgemm_negative_zero_survives_the_k_tail(ops, ta, tb, K):
  """Every product is -2^-160, far below the subnormals, so fmaf(-t, t, +-0) = -0.0 all along the chain: the result is
  -0.0.  A zero product padded onto the tail (fmaf(0, 0, -0) = +0) would turn it into +0.0."""
  M, N = 129, 65
  t = np.float32(2.0 ** -80)
  opA = np.full((M, K), -t, np.float32); opB = np.full((K, N), t, np.float32)
  exp = _ref(opA, opB)
  assert (bits(exp) == 0x80000000).all()
  got = ops.sgemm(cu(_stored(opA, ta)), cu(_stored(opB, tb)), ta, tb)
  assert (bits(got) == 0x80000000).all(), "the K tail of the chain lost the sign of -0.0"


# ================================================================================================
# split-K over the batch: exact Dense and Cross backward
# ================================================================================================
def sgemm_batch_ranges(B):
  """Row ranges of the deterministic split-K (sgemm_batch_splits, then sgemm_split's kps: a multiple of 16)."""
  Z = min(max(cdiv(B, 4096), 1), 16)
  if Z <= 1:
    return [(0, B)]
  kps = cdiv(cdiv(B, Z), 16) * 16
  return [(lo, min(B, lo + kps)) for lo in range(0, B, kps)]


def split_k_ref(a, g, reverse=False):
  """a^T g over the batch as the kernels do it: one fmaf chain per range (oracle.scores on the row slice), the range
  results then summed in fp32 left to right.  `reverse` sums them the other way (for the self-test only)."""
  parts = [orc.scores(np.ascontiguousarray(a[lo:hi].T), np.ascontiguousarray(g[lo:hi].T)) for lo, hi in sgemm_batch_ranges(a.shape[0])]
  if reverse:
    parts = parts[::-1]
  out = parts[0]
  for p in parts[1:]:
    out = out + p          # float32 + float32
  return out


def dense_db_ref(dz):
  """The Dense bias gradient: row splits of ceil(B/64) rows, each summed sequentially in float64, then the partials in
  order (cumsum is sequential; np.sum is pairwise), rounded once to float32."""
  B = dz.shape[0]
  rps = cdiv(B, 64)
  parts = [np.cumsum(dz[lo:lo + rps].astype(np.float64), axis=0)[-1] for lo in range(0, B, rps)]
  return np.cumsum(np.stack(parts), axis=0)[-1].astype(np.float32)


def cross_db_ref(gp):
  """The Cross bias gradient: the same row splits, each summed sequentially in fp32, the partials then in fp32 in order."""
  B = gp.shape[0]
  rps = cdiv(B, 64)
  parts = [np.cumsum(gp[lo:lo + rps], axis=0, dtype=np.float32)[-1] for lo in range(0, B, rps)]
  return np.cumsum(np.stack(parts), axis=0, dtype=np.float32)[-1]


def adversarial_column(B):
  """2^60, then ones, then -2^60: the float64 sum depends on its order (2^60 + 1 rounds back to 2^60)."""
  col = np.ones(B, np.float32)
  col[0] = 2.0 ** 60; col[-1] = -(2.0 ** 60)
  return col


@pytest.mark.parametrize("B", SPLIT_B)
def test_dense_exact_backward_split_k(ops, B):
  K, N = DENSE_BWD_KN
  assert not ops.dense_uses_tc(B, K, N)
  rng = np.random.RandomState(B)
  x = rng.normal(size=(B, K)).astype(np.float32); W = rng.normal(size=(K, N)).astype(np.float32)
  b = rng.normal(size=(N,)).astype(np.float32); g = rng.normal(size=(B, N)).astype(np.float32)
  g[:, 0] = adversarial_column(B)
  tx, tW, tb = (cu(a).requires_grad_(True) for a in (x, W, b))
  y = ops.dense(tx, tW, tb, None)
  y.backward(cu(g))
  assert_bits(tW.grad, split_k_ref(x, g), "dW")
  assert_bits(tb.grad, dense_db_ref(g), "db")
  assert_bits(tx.grad, orc.scores(g, W), "dx")


@pytest.mark.parametrize("B", SPLIT_B)
def test_cross_exact_backward_split_k(ops, B):
  D = CROSS_BWD_D
  rng = np.random.RandomState(B + 1)
  x0 = rng.normal(size=(B, D)).astype(np.float32); x = rng.normal(size=(B, D)).astype(np.float32)
  W = (rng.normal(size=(D, D)) * 0.2).astype(np.float32); b = rng.normal(size=(D,)).astype(np.float32)
  g = rng.normal(size=(B, D)).astype(np.float32)
  t = [cu(a).requires_grad_(True) for a in (x0, x, W, b)]
  out = ops.cross(t[0], t[1], t[2], t[3], 0.0)
  out.backward(cu(g))
  gp = g * x0                                 # one fp32 multiply
  assert_bits(t[2].grad, split_k_ref(x, gp), "dW")
  assert_bits(t[3].grad, cross_db_ref(gp), "db")
  assert_bits(t[1].grad, orc.scores(gp, W) + g, "dx")   # chain + g, diag_scale = 0
  pv = orc.scores(x, W.T) + b                 # prod = chain + bias
  assert_bits(t[0].grad, g * pv, "dx0")


@pytest.mark.parametrize("B,K,N", DENSE_FWD_CASES)
@pytest.mark.parametrize("act", [None, "relu", "sigmoid"])
def test_dense_exact_forward(ops, B, K, N, act):
  assert not ops.dense_uses_tc(B, K, N)
  rng = np.random.RandomState(B * 7 + K + N)
  x = rng.normal(size=(B, K)).astype(np.float32); W = rng.normal(size=(K, N)).astype(np.float32)
  b = rng.normal(size=(N,)).astype(np.float32)
  z = orc.scores(x, W.T) + b                  # chain + bias: one fp32 add
  y = ops.dense(cu(x), cu(W), cu(b), act)
  if act is None:
    assert_bits(y, z)
  elif act == "relu":
    assert_bits(y, np.where(z > 0, z, np.float32(0)))
  else:
    assert_bits(ops.attached_logits(y), z)
    exp = (1.0 / (1.0 + np.exp(-z.astype(np.float64)))).astype(np.float32)
    ulp = np.abs(bits(y).astype(np.int64) - bits(exp).astype(np.int64))
    assert ulp.max() <= SIGMOID_ULP, ulp.max()


# ================================================================================================
# row select: the exact scan, the merges, the MovieLens dense route
# ================================================================================================
def rowselect_cap(k):
  c = 1
  while c < 2 * k:
    c <<= 1
  return max(c, 1024)


def sel_counts(k):
  """Candidate counts per query: k - 1, k, k + 1; cap - 1, cap, cap + 1; several compactions."""
  cap = rowselect_cap(k)
  return sorted({n for n in (k - 1, k, k + 1, cap - 1, cap, cap + 1, SEL_MANY * cap + 17) if n > 0})


TINY = np.float32(2.0 ** -80)


def sel_data(pattern, N, seed):
  """(q [2, 2], corpus [N, 2]).  q = [[1, t], [-1, t]] with t = 2^-80: score = fmaf(t, c1, +-c0), i.e. +-c0, and
  sign(c1) * 0.0 where c0 == 0 (the product underflows), so -0.0 and +0.0 are both real scores.  The second query
  reverses the order of the first."""
  rng = np.random.RandomState(seed)
  c = np.empty((N, 2), np.float32)
  c[:, 1] = np.where(rng.rand(N) < 0.5, -TINY, TINY)
  if pattern == "random":
    c[:, 0] = rng.normal(size=N)
  elif pattern == "ascending":
    c[:, 0] = np.arange(N)                  # every candidate beats the running threshold (query 0) or none does (query 1)
  elif pattern == "equal":
    c[:, 0] = 1.0
    c[:, 1] = TINY
  elif pattern == "inf":
    c[:, 0] = rng.choice(np.array([np.inf, -np.inf, 0.5, -0.5], np.float32), size=N, p=[0.3, 0.3, 0.2, 0.2])
  elif pattern == "zeros":
    c[:, 0] = np.where(rng.rand(N) < 0.7, 0.0, -np.abs(rng.normal(size=N)))
  else:
    raise ValueError(pattern)
  q = np.array([[1.0, TINY], [-1.0, TINY]], np.float32)
  return q, c


def check_scan(ops, q, c, k, index_offset=0, state=None):
  es, ei = orc.topk_scan(q, c, k, index_offset=index_offset, state=state)
  st = None if state is None else (cu(state[0]), cu(state[1]))
  s, i = ops.topk_scan(cu(q), cu(c), k, index_offset=index_offset, state=st)
  assert tuple(s.shape) == es.shape
  np.testing.assert_array_equal(i.cpu().numpy(), ei)
  assert_bits(s, es)
  return es, ei


@pytest.mark.parametrize("k", SEL_K)
@pytest.mark.parametrize("pattern", SEL_PATTERNS)
def test_row_select_counts_and_scores(ops, k, pattern):
  for N in sel_counts(k):
    q, c = sel_data(pattern, N, k * 31 + N)
    es, ei = check_scan(ops, q, c, k, index_offset=1000)
    if pattern == "equal":
      np.testing.assert_array_equal(ei, np.tile(np.arange(1000, 1000 + min(k, N)), (2, 1)))
    if pattern == "zeros" and min(k, N) > 8:   # the first query's list is mostly +-0.0 ties: both signs present, by index
      head = bits(es[0])
      assert (head == 0x80000000).any() and (head == 0).any()


@pytest.mark.parametrize("k", SEL_K)
@pytest.mark.parametrize("delta", [-1, 0, 1])
def test_row_select_compaction_boundary(ops, k, delta):
  """After the first compaction (cap candidates in, k kept) the next slab holds m passing candidates, so the buffer
  holds k + m = 3 cap / 4 + delta: room cap / 4 + 1 and cap / 4 keep filling, cap / 4 - 1 compacts.  Later slabs fail
  the threshold except the last five rows, which win."""
  cap = rowselect_cap(k)
  m = 3 * cap // 4 - k + delta
  assert 0 <= m <= cap - k
  N = 2 * cap + 100
  rng = np.random.RandomState(k + delta)
  v = np.full(N, -5.0, np.float32)
  v[:cap] = rng.uniform(0.0, 1.0, size=cap)          # first slab
  v[cap:cap + m] = rng.uniform(2.0, 3.0, size=m)     # second slab: m above the threshold, the rest below
  v[-5:] = 4.0
  c = np.stack([v, np.full(N, TINY, np.float32)], 1)
  q = np.array([[1.0, TINY]], np.float32)
  es, ei = check_scan(ops, q, c, k)
  w = min(k, 5)
  np.testing.assert_array_equal(ei[0, :w], np.arange(N - 5, N - 5 + w))   # the last rows win, ties by index


@pytest.mark.parametrize("k", [513, 1025, 2048])
def test_row_select_carried_state(ops, k):
  """A carried [Q, w] state (w = 0, < k, = k) from an earlier chunk, merged with this chunk's rows at an offset."""
  cap = rowselect_cap(k)
  rng = np.random.RandomState(k)
  q = rng.normal(size=(3, 8)).astype(np.float32)
  prev = rng.normal(size=(cap + 5, 8)).astype(np.float32)
  c = rng.normal(size=(cap + 1, 8)).astype(np.float32)
  for w in (0, k // 2, k):
    state = None if w == 0 else orc.topk_scan(q, prev, w)
    if state is not None:
      st = (np.ascontiguousarray(state[0][:, ::-1]), np.ascontiguousarray(state[1][:, ::-1]))   # order is not required
    else:
      st = (np.zeros((3, 0), np.float32), np.zeros((3, 0), np.int64))
    check_scan(ops, q, c, k, index_offset=prev.shape[0], state=st)
  # a state of higher indices than the chunk, every score equal: the chunk's lowest indices win the ties
  q2, c2 = sel_data("equal", cap + 1, k)
  for w in (k // 2, k):
    st = (np.repeat(np.array([[1.0], [-1.0]], np.float32), w, 1), np.tile(np.arange(10 ** 6, 10 ** 6 + w), (2, 1)))
    es, ei = check_scan(ops, q2, c2, k, state=st)
    np.testing.assert_array_equal(ei, np.tile(np.arange(k), (2, 1)))


def scan_nc(Q, N):
  """scan_plan's chunk width at the default 256 MB budget."""
  nc = (256 << 20) // (Q * 4) // 128 * 128
  return min(max(nc, 1024), cdiv(max(N, 1), 128) * 128)


def test_exact_scan_chunk_loop(ops):
  """Q large enough that scan_plan cuts N into chunks of >= 1024 columns (a multiple of 128), N not a multiple."""
  Q, N, k = CHUNK_QNK
  nc = scan_nc(Q, N)
  assert 1024 <= nc < N and N % nc
  g = torch.Generator(device="cuda"); g.manual_seed(5)
  q = torch.randn((Q, 4), generator=g, device="cuda"); c = torch.randn((N, 4), generator=g, device="cuda")
  s, i = ops.topk_scan(q, c, k, index_offset=77)
  rows = torch.from_numpy(np.linspace(0, Q - 1, 96).astype(np.int64)).to(dev())
  es, ei = orc.topk_scan(q[rows].cpu().numpy(), c.cpu().numpy(), k, index_offset=77)
  np.testing.assert_array_equal(i[rows].cpu().numpy(), ei)
  assert_bits(s[rows], es)


def state_bytes(Q, k):
  up = lambda x: (x + 255) // 256 * 256
  return up(Q * k * 4) + up(Q * k * 8)


@pytest.mark.parametrize("Q,N,k,extra", SHRINK_CASES)
def test_exact_scan_workspace_shrink(ops, Q, N, k, extra):
  """A workspace above 2 * state_bytes + Q * 4096 but below the plan: the scan cuts smaller chunks instead of failing."""
  from recommenders_b200._ffi import ptr, stream
  d = 8
  fixed = 2 * state_bytes(Q, k)
  ws_bytes = fixed + extra
  assert fixed + Q * 4096 < ws_bytes < ops.lib().tfrs_topk_scan_workspace_bytes(Q, N, d, k)
  rng = np.random.RandomState(Q + N)
  q = rng.normal(size=(Q, d)).astype(np.float32); c = rng.normal(size=(N, d)).astype(np.float32)
  es, ei = orc.topk_scan(q, c, k, index_offset=9)
  ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev())
  s = torch.empty((Q, k), device=dev()); i = torch.empty((Q, k), dtype=torch.int64, device=dev())
  tq, tc_ = cu(q), cu(c)
  rc = ops.lib().tfrs_topk_scan_f32(ptr(tq), Q, ptr(tc_), N, d, k, 9, None, None, 0, ptr(s), ptr(i), ptr(ws), ws_bytes, stream())
  assert rc == 0
  np.testing.assert_array_equal(i.cpu().numpy(), ei)
  assert_bits(s, es)
  # at the bound itself the shrink is not taken: a clean error, nothing launched
  rc = ops.lib().tfrs_topk_scan_f32(ptr(tq), Q, ptr(tc_), N, d, k, 9, None, None, 0, ptr(s), ptr(i), ptr(ws), fixed + Q * 4096,
                                    stream())
  assert rc == -4


def sorted_lists(L, Q, k_in, seed, levels=37):
  """[L, Q, k_in] lists in the total order (score desc, index asc), scores on a coarse grid (many ties across lists),
  indices distinct over all lists."""
  rng = np.random.RandomState(seed)
  s = (rng.randint(0, levels, size=(L, Q, k_in)) - levels // 2).astype(np.float32) * np.float32(0.25)
  s[rng.rand(L, Q, k_in) < 0.05] = -np.inf
  idx = np.stack([rng.permutation(L * k_in) for _ in range(Q)], 1).reshape(Q, L, k_in).transpose(1, 0, 2).astype(np.int64)
  order = np.lexsort((idx, -s.astype(np.float64)), axis=-1)
  return np.take_along_axis(s, order, -1), np.take_along_axis(idx, order, -1)


@pytest.mark.parametrize("L,k_in,k_out", SORT_MERGE_CASES + TREE_MERGE_CASES)
def test_list_merges(ops, L, k_in, k_out):
  """Both merges equal the oracle's: the sorting merge (row select over n_lists * k_in candidates) and the tree merge
  of sorted lists, at and beyond its limits (more than MS_MAX_LISTS lists, a level larger than 160 KB), where it hands
  over to the sorting merge."""
  s, i = sorted_lists(L, 3, k_in, L * 10000 + k_in)
  es, ei = orc.topk_merge(s, i, k_out)
  for sorted_flag in (False, True):
    ms, mi = ops.topk_merge(cu(s), cu(i), k_out, sorted_lists=sorted_flag)
    np.testing.assert_array_equal(mi.cpu().numpy(), ei, err_msg=f"sorted_lists={sorted_flag}")
    assert_bits(ms, es, f"sorted_lists={sorted_flag}")


def test_merge_of_unsorted_lists_past_cap(ops):
  """The sorting merge takes lists in any order."""
  rng = np.random.RandomState(3)
  L, Q, k_in, k_out = 3, 4, 1500, 2048
  s = (rng.randint(0, 9, size=(L, Q, k_in)).astype(np.float32) - 4) * np.float32(0.5)
  i = rng.permutation(L * Q * k_in).reshape(L, Q, k_in).astype(np.int64)
  es, ei = orc.topk_merge(s, i, k_out)
  ms, mi = ops.topk_merge(cu(s), cu(i), k_out)
  np.testing.assert_array_equal(mi.cpu().numpy(), ei)
  assert_bits(ms, es)


@pytest.mark.parametrize("k_out", [512, 1025, 2048])
def test_merge_ties_arriving_after_the_threshold(ops, k_out):
  """Every score equal, the first list holding the higher indices: the threshold is set on first-list entries, and the
  second list's entries, arriving later with the same score and lower indices, must still get in."""
  k_in = 1500
  s = np.full((2, 2, k_in), 0.75, np.float32)
  i = np.stack([np.tile(np.arange(10 ** 6, 10 ** 6 + k_in), (2, 1)), np.tile(np.arange(k_in), (2, 1))]).astype(np.int64)
  es, ei = orc.topk_merge(s, i, k_out)
  np.testing.assert_array_equal(ei[:, :min(k_out, k_in)], np.tile(np.arange(min(k_out, k_in)), (2, 1)))
  for sorted_flag in (False, True):
    ms, mi = ops.topk_merge(cu(s), cu(i), k_out, sorted_lists=sorted_flag)
    np.testing.assert_array_equal(mi.cpu().numpy(), ei, err_msg=f"sorted_lists={sorted_flag}")
    assert_bits(ms, es)


def test_movielens_dense_route_at_k_1025(ops):
  import movielens_eval_oracle as mlo
  rng = np.random.RandomState(1025)
  Q, N, d, k = 6, 5000, 16, OVERRIDE_K
  q = rng.normal(size=(Q, d)).astype(np.float32); c = rng.normal(size=(N, d)).astype(np.float32)
  lens = np.array([0, 1, 40, 1500, 7, 300])
  rows = np.concatenate([np.sort(rng.choice(N, size=n, replace=False)) for n in lens]).astype(np.int64)
  off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
  es, ei = mlo.topk_overriding(q, c, k, off, rows)
  s, i = ops.topk_overriding_dense(cu(q), cu(c), k, off, rows)
  np.testing.assert_array_equal(i.cpu().numpy(), ei)
  assert_bits(s, es)


# ================================================================================================
# tensor-core top-K on a corpus that starts off a 16-byte boundary
# ================================================================================================
def _unaligned(c, off):
  flat = torch.zeros(off + c.size + 4, device=dev())
  v = flat[off:off + c.size].view(c.shape)
  v.copy_(cu(c))
  assert v.data_ptr() % 16 == 4 * off
  return v


@pytest.fixture(scope="module", params=TC_UNALIGNED_D)
def tc_data(request):
  Q, N, k = TC_QNK
  d = request.param
  rng = np.random.RandomState(d)
  q = rng.normal(size=(Q, d)).astype(np.float32); c = rng.normal(size=(N, d)).astype(np.float32)
  return q, c, k, orc.scores(q, c)


def _exp_topk(S, k):
  order = np.lexsort((np.broadcast_to(np.arange(S.shape[1]), S.shape), -S.astype(np.float64)), axis=1)[:, :k]
  return np.take_along_axis(S, order, 1), order


@pytest.mark.parametrize("off", TC_UNALIGNED_OFF)
def test_tc_topk_unaligned_corpus(ops, tc_data, off):
  q, c, k, S = tc_data
  Q, d = q.shape; N = c.shape[0]
  assert ops.uses_tc_scan(Q, N, d, k)
  es, ei = orc.topk_scan(q, c, k)
  cu_c = cu(c)
  image = ops.index_build(cu_c)
  a_s, a_i = ops.topk(cu(q), cu_c, k, image=image)
  np.testing.assert_array_equal(a_i.cpu().numpy(), ei); assert_bits(a_s, es)
  uc = _unaligned(c, off)
  assert ops.tc_corpus(uc).data_ptr() % 16 == 0
  for img in (image, "anchor_unaligned"):       # a prebuilt image, and one built from the unaligned corpus
    s, i = ops.topk(cu(q), uc, k, image=img)
    np.testing.assert_array_equal(i.cpu().numpy(), ei); assert_bits(s, es)
  s, i = ops.topk_tc(cu(q), uc, image, k, index_offset=5)
  np.testing.assert_array_equal(i.cpu().numpy(), ei + 5); assert_bits(s, es)
  # exclusions: over-fetch k + E, drop the excluded ids
  E = 4
  ex = np.stack([ei[:, 0], ei[:, 3], np.full(Q, N - 1), ei[:, k - 1]], 1).astype(np.int64)
  fs, fi = orc.topk_scan(q, c, k + E)
  xs, xi = orc.exclude(fs, fi, ex, k)
  for corpus in (cu_c, uc):
    s, i = ops.topk_tc_exclude(cu(q), corpus, image, k, cu(ex))
    np.testing.assert_array_equal(i.cpu().numpy(), xi); assert_bits(s, xs)
  # count mode: positives at scores of the corpus, so ties with them are exercised
  pos = S[np.arange(Q), (np.arange(Q) * 97) % N].astype(np.float32)
  ecount = np.minimum(k, (S > pos[:, None]).sum(1)).astype(np.int32)
  for corpus in (cu_c, uc):
    np.testing.assert_array_equal(ops.topk_tc_count(cu(q), corpus, image, k, cu(pos)).cpu().numpy(), ecount)


def test_tc_streaming_unaligned_chunk(ops, tc_data):
  import recommenders_b200 as tfrs
  q, c, k, _ = tc_data
  es, ei = orc.topk_scan(q, c, k)
  layer = tfrs.layers.factorized_top_k.Streaming(k=k).index_from_dataset([_unaligned(c, 3)])
  s, i = layer(cu(q))
  np.testing.assert_array_equal(i.cpu().numpy().astype(np.int64), ei); assert_bits(s, es)


def test_tc_copies_only_when_needed(ops):
  a = torch.zeros((100, 36), device=dev())
  assert ops.tc_corpus(a) is a
  odd = torch.zeros(1 + 100 * 33, device=dev())[1:].view(100, 33)   # d % 4 != 0: scalar loads, no copy
  assert ops.tc_corpus(odd) is odd
  un = torch.zeros(1 + 100 * 36, device=dev())[1:].view(100, 36)
  cp = ops.tc_corpus(un)
  assert cp is not un and cp.data_ptr() % 16 == 0 and torch.equal(cp, un)


@pytest.mark.parametrize("off", TC_UNALIGNED_OFF)
def test_tc_c_abi_rejects_unaligned_corpus(ops, tc_data, off):
  """The C entry points refuse the pointer before anything is launched."""
  from recommenders_b200._ffi import last_error, ptr, stream
  q, c, k, _ = tc_data
  Q, d = q.shape; N = c.shape[0]
  cu_c = cu(c)
  image = ops.index_build(cu_c)
  uc = _unaligned(c, off)
  tq = cu(q)
  wsb = max(ops.lib().tfrs_topk_tc_workspace_bytes(Q, N, d, kk) for kk in (k, k + 2))
  ws = torch.empty(wsb, dtype=torch.uint8, device=dev())
  s = torch.full((Q, k), 7.0, device=dev()); i = torch.full((Q, k), -3, dtype=torch.int64, device=dev())
  cnt = torch.full((Q,), -3, dtype=torch.int32, device=dev()); pos = torch.zeros(Q, device=dev())
  ex = torch.zeros((Q, 2), dtype=torch.int64, device=dev())
  lib = ops.lib()
  rcs = [lib.tfrs_topk_tc_f32(ptr(tq), Q, ptr(uc), ptr(image), N, d, k, 0, ptr(s), ptr(i), ptr(ws), ws.numel(), stream()),
         lib.tfrs_topk_tc_exclude_f32(ptr(tq), Q, ptr(uc), ptr(image), N, d, k, 0, None, ptr(ex), 2, ptr(s), ptr(i), ptr(ws),
                                      ws.numel(), stream()),
         lib.tfrs_topk_tc_count_f32(ptr(tq), Q, ptr(uc), ptr(image), N, d, k, ptr(pos), ptr(cnt), ptr(ws), ws.numel(), stream())]
  for rc in rcs:
    assert rc == -1
  assert "16-byte aligned" in last_error()
  torch.cuda.synchronize()
  assert (s == 7.0).all() and (i == -3).all() and (cnt == -3).all()   # nothing was written
