"""Edge cases of the split-fp16 tensor-core GEMM (csrc/split_gemm.cu, operand images from csrc/tc_split.cuh) behind
tfrs_gemm_tc_f32, the full-rank and low-rank Cross and the Dense layer: shape, stride, chunk and scheduling edges of
every epilogue, long single accumulation chains (full-rank Cross wider than 1024), the whole fp32 exponent range, and
non-finite inputs.

The reference is NumPy float64 of the same formula.  Bars (DESIGN section 2):
  (T) max |got - ref| <= 1e-5 * max |ref|, per tensor;
  (E) per element, |got - ref| <= 1e-5 (|A| |B|)_ij + 2^-36 (amax_A sum_k |B_kj| + amax_B sum_k |A_ik|), amax over the
      finite entries; epilogues add 2^-22 of the magnitude of each term they add after the product;
  (B) bitwise.
"""
import ctypes

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

SENTINEL = 0x7FC01234        # a NaN with a payload: padding that a kernel overwrites cannot keep these bits by accident
FLT_MAX = float(np.finfo(np.float32).max)
FLT_MIN = float(np.finfo(np.float32).tiny)


@pytest.fixture(scope="module")
def ops():
  from recommenders_b200 import ops as o
  return o


def _rand(shape, seed, scale=1.0):
  g = torch.Generator(device="cuda"); g.manual_seed(seed)
  return torch.randn(shape, generator=g, device="cuda") * scale


def _rand_away_from_zero(shape, seed):
  """Unit normal data whose entries all have |v| >= 2^-10: every 2^s-scaled copy with s in [-116, 124] is exact."""
  v = _rand(shape, seed)
  return torch.where(v.abs() < 2.0 ** -10, torch.copysign(torch.full_like(v, 2.0 ** -10), v), v)


def _sc(v, e):
  return v * (2.0 ** e)


def _f64(t):
  return t.detach().cpu().numpy().astype(np.float64)


def _bits(t):
  return t.detach().contiguous().view(torch.int32).cpu()


def _sentinel_like(rows, cols):
  return torch.full((rows, cols), SENTINEL, dtype=torch.int32, device="cuda").view(torch.float32)


def _ratio_T(got, ref):
  got = np.asarray(got, np.float64); ref = np.asarray(ref, np.float64)
  return float(np.abs(got - ref).max() / (1e-5 * np.abs(ref).max()))


def _T(got, ref, what):
  r = _ratio_T(got, ref)
  assert r <= 1.0, f"{what}: max |err| is {r:.3f} x the (T) bar 1e-5 * max|ref|"
  return r


def _ebar(A, B):
  """Bar (E) for A [M,K] . B [K,N] (float64 op forms); non-finite entries count as 0 (the rescale ignores them)."""
  Af = np.where(np.isfinite(A), np.abs(A), 0.0); Bf = np.where(np.isfinite(B), np.abs(B), 0.0)
  return 1e-5 * (Af @ Bf) + 2.0 ** -36 * (Af.max() * Bf.sum(0)[None, :] + Bf.max() * Af.sum(1)[:, None])


def _E(got, ref, tol, what, check=None):
  """Per-element bar (E) where `check` (default: everywhere); where ref overflows fp32, got must be non-finite."""
  got = np.asarray(got, np.float64)
  check = np.ones(ref.shape, bool) if check is None else check
  over = check & ~(np.abs(ref) <= FLT_MAX)
  assert not np.isfinite(got[over]).any(), f"{what}: a finite result where fp32 overflows"
  m = check & ~over
  assert np.isfinite(got[m]).all(), f"{what}: {int((~np.isfinite(got[m])).sum())} non-finite results where fp32 is finite"
  err = np.abs(got - ref)
  bad = m & (err > tol)
  if bad.any():
    i = np.argwhere(bad)[0]
    raise AssertionError(f"{what}: {int(bad.sum())} elements miss bar (E); first {tuple(i)}: got {got[tuple(i)]!r} "
                         f"ref {ref[tuple(i)]!r} err {err[tuple(i)]:.3e} bar {tol[tuple(i)]:.3e}")


# ------------------------------------------------------------------------------------------------
# tfrs_gemm_tc_f32 through the C ABI: C[M,N] = opA(A) . opB(B), strides and workspace of our own
# ------------------------------------------------------------------------------------------------
def _operands(ta, tb, M, N, K, seed, pad_a=0, pad_b=0, make=None):
  """Stored A ([K, M + pad] when transposed, else [M, K + pad]) and B ([N, K + pad] when transposed, else [K, N + pad])."""
  make = make or (lambda shape, s: _rand(shape, s))
  A = make((K, M + pad_a) if ta else (M, K + pad_a), seed)
  Bm = make((N, K + pad_b) if tb else (K, N + pad_b), seed + 1)
  return A, Bm


def _op64(ta, tb, M, N, K, A, Bm):
  a = _f64(A); b = _f64(Bm)
  return (a[:, :M].T if ta else a[:, :K]), (b[:, :K].T if tb else b[:, :N])


def _ws(ops, M, N, K, fill=None):
  ws = torch.empty(ops.lib().tfrs_gemm_tc_workspace_bytes(M, N, K), dtype=torch.uint8, device="cuda")
  if fill is not None:
    ws.fill_(fill)
  return ws


def _gemm(ops, ta, tb, M, N, K, A, Bm, pad_c=0, ws=None, ws_bytes=None, ws_offset=0):
  """One tfrs_gemm_tc_f32 call; returns C [M, N + pad_c] (padding pre-filled with SENTINEL)."""
  C = _sentinel_like(M, N + pad_c)
  ws = _ws(ops, M, N, K) if ws is None else ws
  ops.check(ops.lib().tfrs_gemm_tc_f32(int(ta), int(tb), M, N, K, ops.ptr(A), A.stride(0), ops.ptr(Bm), Bm.stride(0), ops.ptr(C),
                                       C.stride(0), ctypes.c_void_p(ws.data_ptr() + ws_offset),
                                       ws.numel() - ws_offset if ws_bytes is None else ws_bytes, ops.stream()), "gemm_tc")
  return C


TRANS = [(False, False), (False, True), (True, False), (True, True)]
_MS, _NS, _KS = [1, 255, 256, 257], [1, 127, 128, 129], [1, 15, 16, 17, 63, 64, 65]
COVER = [(_MS[i % 4], _NS[(i + 2) % 4], _KS[i]) for i in range(7)]   # every M, N and K value, each with every transposition


@pytest.mark.parametrize("ta,tb", TRANS)
@pytest.mark.parametrize("M,N,K", COVER)
def test_gemm_shape_edges(ops, M, N, K, ta, tb):
  A, Bm = _operands(ta, tb, M, N, K, 11)
  a, b = _op64(ta, tb, M, N, K, A, Bm)
  C = _gemm(ops, ta, tb, M, N, K, A, Bm)
  _T(_f64(C), a @ b, f"gemm {M}x{N}x{K} ta={ta} tb={tb}")
  _E(_f64(C), a @ b, _ebar(a, b), "gemm (E)")


@pytest.mark.parametrize("ta,tb", TRANS)
@pytest.mark.parametrize("K", [1024, 1025, 2048, 2049])
def test_gemm_chunk_edges(ops, K, ta, tb):
  """K = 1024 is one chain of 16 slabs; 1025 adds a chunk of one slab holding one live index; 2048 / 2049 likewise."""
  M, N = 300, 200
  A, Bm = _operands(ta, tb, M, N, K, 13)
  a, b = _op64(ta, tb, M, N, K, A, Bm)
  C = _gemm(ops, ta, tb, M, N, K, A, Bm)
  _T(_f64(C), a @ b, f"gemm K={K} ta={ta} tb={tb}")
  _E(_f64(C), a @ b, _ebar(a, b), "gemm (E)")


def _sms():
  return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


@pytest.mark.parametrize("case", ["odd_slabs_items", "odd_last_chunk"])
def test_gemm_several_items_per_cta_with_odd_slab_counts(ops, case):
  """The 2-stage ring's stage and phase carry over item boundaries: with an odd slab count per item they flip between
  items.  (a) 2*SMs + 1 items of 3 slabs each; (b) chunked, per_chunk * n_kc > SMs, last chunk of 5 slabs."""
  sms = _sms()
  if case == "odd_slabs_items":
    M, N, K = 256 * (2 * sms + 1), 128, 192
  else:
    M, N, K = 1024, 1024, 64 * (16 * 4 + 5)
    assert (M // 256) * (N // 128) * 5 > sms
  A, Bm = _operands(False, True, M, N, K, 17)
  a, b = _op64(False, True, M, N, K, A, Bm)
  C = _gemm(ops, False, True, M, N, K, A, Bm)
  _T(_f64(C), a @ b, case)


@pytest.mark.parametrize("ta,tb", TRANS)
@pytest.mark.parametrize("M,N,K,pad", [(257, 129, 65, 3), (300, 200, 1100, 37)])
def test_gemm_strides_and_padding_untouched(ops, M, N, K, pad, ta, tb):
  A, Bm = _operands(ta, tb, M, N, K, 19, pad_a=pad, pad_b=pad + 2)
  a, b = _op64(ta, tb, M, N, K, A, Bm)
  C = _gemm(ops, ta, tb, M, N, K, A, Bm, pad_c=pad + 4)
  _T(_f64(C[:, :N]), a @ b, f"strided gemm pad={pad}")
  assert (_bits(C[:, N:]) == SENTINEL).all(), "C's padding columns were written"


@pytest.mark.parametrize("ta,tb", [(False, True), (True, False)])
@pytest.mark.parametrize("K", [300, 2100])
def test_gemm_garbage_workspace(ops, K, ta, tb):
  """A workspace full of 0xFF bytes (NaN floats, ~0 statistics) gives the same bits as a zeroed one: the images, the
  statistics and the partials are fully rewritten by every call."""
  M, N = 333, 257
  A, Bm = _operands(ta, tb, M, N, K, 23)
  c0 = _gemm(ops, ta, tb, M, N, K, A, Bm, ws=_ws(ops, M, N, K, 0))
  c1 = _gemm(ops, ta, tb, M, N, K, A, Bm, ws=_ws(ops, M, N, K, 0xFF))
  assert torch.equal(_bits(c0), _bits(c1))


def test_gemm_argument_checks(ops):
  M, N, K = 300, 200, 100
  A, Bm = _operands(False, False, M, N, K, 29)
  C = torch.empty((M, N), device="cuda")
  ws = _ws(ops, M, N, K)
  lib = ops.lib()

  def call(ta, tb, lda, ldb, ws_ptr, ws_bytes):
    ops.check(lib.tfrs_gemm_tc_f32(ta, tb, M, N, K, ops.ptr(A), lda, ops.ptr(Bm), ldb, ops.ptr(C), N, ws_ptr, ws_bytes,
                                   ops.stream()), "gemm_tc")

  good = ctypes.c_void_p(ws.data_ptr())
  call(0, 0, K, N, good, ws.numel())
  for ta, tb, lda, ldb, what in [(0, 0, K - 1, N, "lda"), (1, 0, M - 1, N, "lda"), (0, 0, K, N - 1, "ldb"),
                                 (0, 1, K, K - 1, "ldb")]:
    with pytest.raises(ValueError, match="lda|ldb"):
      call(ta, tb, lda, ldb, good, ws.numel())
  with pytest.raises(RuntimeError, match="workspace too small"):
    call(0, 0, K, N, good, ws.numel() - 1)
  big = torch.empty(ws.numel() + 16, dtype=torch.uint8, device="cuda")
  with pytest.raises(ValueError, match="16-byte aligned"):
    call(0, 0, K, N, ctypes.c_void_p(big.data_ptr() + 4), ws.numel())


# ------------------------------------------------------------------------------------------------
# DENSE: y = act(x . W + b), through ops.dense, forward and backward
# ------------------------------------------------------------------------------------------------
def _dense_case(ops, B, K, N, act, seed, bias=True, xs=None):
  x = _rand((B, K), seed) if xs is None else xs
  W = _rand((K, N), seed + 1, K ** -0.5); b = _rand((N,), seed + 2, 0.1) if bias else None
  gy = _rand((B, N), seed + 3)
  xg, Wg = x.clone().requires_grad_(True), W.clone().requires_grad_(True)
  bg = None if b is None else b.clone().requires_grad_(True)
  y = ops.dense(xg, Wg, bg, act)
  logits = ops.attached_logits(y) if act == "sigmoid" else None
  logits = None if logits is None else logits.detach().clone()
  y.backward(gy)
  return x, W, b, gy, y.detach(), logits, xg.grad, Wg.grad, None if bg is None else bg.grad


def _dense_check(x, W, b, gy, y, logits, dx, dW, db, act, what):
  x64, W64, g64 = _f64(x), _f64(W), _f64(gy)
  z = x64 @ W64 + (0.0 if b is None else _f64(b))
  y64 = _f64(y)
  if act == "relu":
    # the mask may flip only where |z| is inside the bar: elsewhere it must agree with float64
    sure = np.abs(z) > 1e-5 * np.abs(z).max()
    assert np.array_equal((y64 > 0)[sure], (z > 0)[sure]), f"{what}: relu mask differs away from the kink"
    _T(y64, np.maximum(z, 0), f"{what} y")
    dz = g64 * (y64 > 0)              # gradients through the kernel's own mask
  elif act == "sigmoid":
    s = 1.0 / (1.0 + np.exp(-z))
    _T(y64, s, f"{what} y")
    assert logits is not None, f"{what}: the sigmoid output carries no logits"
    _T(_f64(logits), z, f"{what} logits")
    dz = g64 * y64 * (1.0 - y64)      # the backward works from the saved output
  else:
    _T(y64, z, f"{what} y")
    dz = g64
  _T(_f64(dx), dz @ W64.T, f"{what} dx")
  _T(_f64(dW), x64.T @ dz, f"{what} dW")
  if b is not None:
    _T(_f64(db), dz.sum(0), f"{what} db")


@pytest.mark.parametrize("B", [1023, 1024])
@pytest.mark.parametrize("K", [63, 64])
@pytest.mark.parametrize("N", [63, 64])
def test_dense_routing_edges(ops, B, K, N):
  act = ["relu", None, "sigmoid"][(B + K + N) % 3]
  assert ops.dense_uses_tc(B, K, N) == (B >= 1024 and K >= 64 and N >= 64)
  r = _dense_case(ops, B, K, N, act, 31)
  _dense_check(*r, act, f"dense B={B} K={K} N={N} {act}")


@pytest.mark.parametrize("act", [None, "relu", "sigmoid"])
@pytest.mark.parametrize("K", [1024, 1025, 2049])
def test_dense_chunk_edges(ops, K, act):
  """K > 1024 runs the chunked partials and sg_reduce_chunks_dense_kernel, which applies bias, activation and logits."""
  r = _dense_case(ops, 1024, K, 128, act, 37)
  _dense_check(*r, act, f"dense K={K} {act}")


@pytest.mark.parametrize("K", [256, 1500])
def test_dense_without_bias(ops, K):
  r = _dense_case(ops, 1024, K, 96, "relu", 41, bias=False)
  _dense_check(*r, "relu", f"dense K={K} no bias")


# ------------------------------------------------------------------------------------------------
# CROSS and DX through tfrs_cross_tc_fwd_f32 / _bwd_f32 with a padded row stride
# ------------------------------------------------------------------------------------------------
def _cross_fwd_raw(ops, x0, x, W, b, B, D, ld, diag, x_amax=None, ws_fill=None):
  out, prod = _sentinel_like(B, ld), _sentinel_like(B, ld)
  amax = torch.zeros((1,), dtype=torch.int32, device="cuda")
  ws = torch.empty(ops.lib().tfrs_cross_tc_workspace_bytes(B, D), dtype=torch.uint8, device="cuda")
  if ws_fill is not None:
    ws.fill_(ws_fill)
  ops.check(ops.lib().tfrs_cross_tc_fwd_f32(ops.ptr(x0), ops.ptr(x), ops.ptr(W), ops.ptr(b), B, D, ld, ops.c_f(diag), ops.ptr(out),
                                            ops.ptr(prod), ops.ptr(x_amax), ops.ptr(amax), ops.ptr(ws), ws.numel(), ops.stream()),
            "cross_tc_fwd")
  return out, prod, amax


def _cross_bwd_raw(ops, x0, x, W, prod, g, B, D, ld, diag):
  dx0, dx = _sentinel_like(B, ld), _sentinel_like(B, ld)
  dW = torch.empty((D, D), device="cuda"); db = torch.empty((D,), device="cuda")
  ws = torch.empty(ops.lib().tfrs_cross_tc_bwd_workspace_bytes(B, D), dtype=torch.uint8, device="cuda")
  ops.check(ops.lib().tfrs_cross_tc_bwd_f32(ops.ptr(x0), ops.ptr(x), ops.ptr(W), ops.ptr(prod), ops.ptr(g), B, D, ld, ops.c_f(diag),
                                            ops.ptr(dx0), ops.ptr(dx), ops.ptr(dW), ops.ptr(db), ops.ptr(ws), ws.numel(),
                                            ops.stream()), "cross_tc_bwd")
  return dx0, dx, dW, db


def _cross_ref(x0, x, W, b, g, diag):
  x0, x, W, g = (np.asarray(t, np.float64) for t in (x0, x, W, g))
  prod = x @ W + (0.0 if b is None else np.asarray(b, np.float64)) + diag * x
  gp = g * x0
  return {"out": x0 * prod + x, "prod": prod, "dx0": g * prod, "dx": gp @ W.T + diag * gp + g, "dW": x.T @ gp, "db": gp.sum(0)}


@pytest.mark.parametrize("diag,bias", [(0.0, True), (0.5, True), (0.5, False)])
@pytest.mark.parametrize("B,D", [(1100, 200), (1024, 1024), (1024, 1100)])
def test_cross_padded_stride_fwd_bwd(ops, B, D, diag, bias):
  """D = 1024 is the widest single-launch CROSS / DX; D = 1100 takes the chunk partials and the reduction's epilogue."""
  ld = D + 3
  x0 = _rand((B, ld), 51, 0.5); x = _rand((B, ld), 52, 0.5); g = _rand((B, ld), 53)
  W = _rand((D, D), 54, D ** -0.5); b = _rand((D,), 55, 0.1) if bias else None
  out, prod, amax = _cross_fwd_raw(ops, x0, x, W, b, B, D, ld, diag)
  dx0, dx, dW, db = _cross_bwd_raw(ops, x0, x, W, prod, g, B, D, ld, diag)
  ref = _cross_ref(_f64(x0)[:, :D], _f64(x)[:, :D], _f64(W), None if b is None else _f64(b), _f64(g)[:, :D], diag)
  for name, t in [("out", out), ("prod", prod), ("dx0", dx0), ("dx", dx)]:
    _T(_f64(t[:, :D]), ref[name], f"cross {name} B={B} D={D} diag={diag}")
    assert (_bits(t[:, D:]) == SENTINEL).all(), f"{name}: padding columns were written"
  _T(_f64(dW), ref["dW"], "cross dW")
  _T(_f64(db), ref["db"], "cross db")
  assert int(amax.item()) == int(out[:, :D].abs().max().view(torch.int32).item()), "out_amax is not max |out|"


@pytest.mark.parametrize("B", [1023, 1024])
@pytest.mark.parametrize("D", [63, 64])
def test_cross_routing_edges(ops, B, D):
  x0 = _rand((B, D), 61, 0.5); x = _rand((B, D), 62, 0.5); g = _rand((B, D), 63)
  W = _rand((D, D), 64, D ** -0.5); b = _rand((D,), 65, 0.1)
  ts = [t.clone().requires_grad_(True) for t in (x0, x, W, b)]
  out = ops.cross(*ts, 0.25)
  assert hasattr(out, "_tfrs_amax") == (B >= 1024 and D >= 64)   # attached on the tensor-core path only
  out.backward(g)
  ref = _cross_ref(_f64(x0), _f64(x), _f64(W), _f64(b), _f64(g), 0.25)
  _T(_f64(out), ref["out"], "out")
  for t, name in zip(ts, ["dx0", "dx", "dW", "db"]):
    _T(_f64(t.grad), ref[name], name)


@pytest.mark.parametrize("p", [1, 15, 16, 17, 1024])
@pytest.mark.parametrize("D", [64, 1024, 1025])
def test_cross_lowrank_edges(ops, D, p):
  """D = 1025 is outside cross_lowrank_supported: the layer runs its unfused path, which must be just as right."""
  import recommenders_b200 as tfrs
  B = 1024
  layer = tfrs.layers.dcn.Cross(projection_dim=p, diag_scale=0.5)
  x0 = _rand((B, D), 71, 0.5); x = _rand((B, D), 72, 0.5); g = _rand((B, D), 73)
  xs0, xs = x0.clone().requires_grad_(True), x.clone().requires_grad_(True)
  out = layer(xs0, xs)
  out.backward(g)
  U, V, b = _f64(layer.kernel_u), _f64(layer.kernel_v), _f64(layer.bias)
  x0_, x_, g_ = _f64(x0), _f64(x), _f64(g)
  t = x_ @ U
  prod = t @ V + b + 0.5 * x_
  gp = g_ * x0_
  dt = gp @ V.T
  _T(_f64(out), x0_ * prod + x_, f"lowrank out D={D} p={p}")
  _T(_f64(xs0.grad), g_ * prod, "lowrank dx0")
  _T(_f64(xs.grad), dt @ U.T + 0.5 * gp + g_, "lowrank dx")
  _T(_f64(layer.kernel_u.grad), x_.T @ dt, "lowrank dU")
  _T(_f64(layer.kernel_v.grad), t.T @ gp, "lowrank dV")
  _T(_f64(layer.bias.grad), gp.sum(0), "lowrank db")


# ------------------------------------------------------------------------------------------------
# Long chains: full-rank Cross wider than 1024
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("D", [1024, 1025, 2048, 4096])
def test_cross_long_reduction(ops, D):
  """Forward and every gradient against float64 at B = 1024.  out, prod-based dx0 and dx are checked on 256 sampled rows
  plus the last 128 (the last row tile), dW and db in full.

  With CROSS and DX as one accumulation chain over K = D, an H100 80GB HBM3 measured these errors, as fractions of bar (T):
    D = 1024: out 0.274, dx0 0.354, dx 0.168      D = 2048: out 0.656, dx0 0.711, dx 0.248
    D = 1025: out 0.301, dx0 0.329, dx 0.156      D = 4096: out 1.349, dx0 1.179, dx 0.567
  so K > 1024 now runs in chunks of 1024 for these epilogues too (dW, a PLAIN product over the batch, was chunked already:
  0.46 - 0.51 at every D).  With the chunks, the same card measured out 0.299 / 0.294 / 0.335 and dx0 0.329 / 0.383 /
  0.340 at D = 1025 / 2048 / 4096 (D = 1024 is unchanged)."""
  B = 1024
  x0 = _rand((B, D), 81, 0.5); x = _rand((B, D), 82, 0.5); g = _rand((B, D), 83)
  W = _rand((D, D), 84, D ** -0.5); b = _rand((D,), 85, 0.1)
  ts = [t.clone().requires_grad_(True) for t in (x0, x, W, b)]
  out = ops.cross(*ts, 0.5)
  out.backward(g)
  rows = np.union1d(np.random.RandomState(D).choice(B - 128, 256, replace=False), np.arange(B - 128, B))
  x0_, x_, g_, W_ = _f64(x0), _f64(x), _f64(g), _f64(W)
  prod = x_[rows] @ W_ + _f64(b) + 0.5 * x_[rows]
  gp = g_ * x0_
  r = {"out": _ratio_T(_f64(out)[rows], x0_[rows] * prod + x_[rows]),
       "dx0": _ratio_T(_f64(ts[0].grad)[rows], g_[rows] * prod),
       "dx": _ratio_T(_f64(ts[1].grad)[rows], gp[rows] @ W_.T + 0.5 * gp[rows] + g_[rows]),
       "dW": _ratio_T(_f64(ts[2].grad), x_.T @ gp),
       "db": _ratio_T(_f64(ts[3].grad), gp.sum(0))}
  msg = f"D={D}: error / (T) bar = " + ", ".join(f"{k} {v:.3f}" for k, v in r.items())
  print(msg)
  assert max(r.values()) <= 1.0, msg


# ------------------------------------------------------------------------------------------------
# The fp32 exponent range
# ------------------------------------------------------------------------------------------------
def _normal(t):
  a = t.abs()
  return (a >= FLT_MIN) & (a <= FLT_MAX)


def _assert_scaled_bits(got, base, e, what):
  """got == ldexp(base, e) bit for bit wherever that is a normal fp32 number."""
  want = torch.ldexp(base.double(), torch.tensor(float(e), dtype=torch.float64, device=base.device))
  m = _normal(want)
  assert m.float().mean() > 0.25, f"{what}: too few normal results to compare"
  w32 = want.float()
  diff = (_bits(got)[m.cpu()] != _bits(w32)[m.cpu()])
  assert not diff.any(), f"{what}: {int(diff.sum())} of {int(m.sum())} normal results differ from the unscaled call x 2^{e}"


ST_GEMM = [(-116, 0), (0, -116), (124, -20), (-20, 124), (60, 60), (-60, 50), (-64, -64), (-64, -65), (-65, -65), (-65, -66),
           (-100, -31), (100, 20)]


@pytest.mark.parametrize("ta,tb", [(False, False), (True, True)])
def test_gemm_scale_equivariance(ops, ta, tb):
  """The rescale is an exact power of two, so gemm(2^s A, 2^t B) = 2^(s+t) gemm(A, B) wherever the result is normal --
  including s + t in [-131, -128], where 2^-(exp_a + exp_b) is not a normal float."""
  M, N, K = 300, 200, 1024
  A, Bm = _operands(ta, tb, M, N, K, 91, make=_rand_away_from_zero)
  base = _gemm(ops, ta, tb, M, N, K, A, Bm)
  for s, t in ST_GEMM:
    _assert_scaled_bits(_gemm(ops, ta, tb, M, N, K, _sc(A, s), _sc(Bm, t)), base, s + t, f"gemm s={s} t={t}")


def test_gemm_scale_equivariance_chunked(ops):
  """Chunked K: bitwise where the partials stay normal; at s + t in [-131, -128] the chunk partials (fp32 numbers in the
  output's scale) can be subnormal, so there each result meets bar (E) plus one subnormal rounding (2^-149) per partial,
  and most results are nonzero normal numbers."""
  M, N, K = 256, 256, 4096
  A, Bm = _operands(False, True, M, N, K, 93, make=_rand_away_from_zero)
  base = _gemm(ops, False, True, M, N, K, A, Bm)
  for s, t in [(-116, 0), (60, 60), (-60, -50), (100, 20)]:
    _assert_scaled_bits(_gemm(ops, False, True, M, N, K, _sc(A, s), _sc(Bm, t)), base, s + t, f"chunked gemm s={s} t={t}")
  for s, t in [(-64, -64), (-65, -65), (-65, -66)]:
    As, Bs = _sc(A, s), _sc(Bm, t)
    got = _f64(_gemm(ops, False, True, M, N, K, As, Bs))
    a, b = _op64(False, True, M, N, K, As, Bs)
    ref = a @ b
    assert (np.abs(ref) >= FLT_MIN).mean() > 0.5 and (np.abs(got) >= FLT_MIN).mean() > 0.5, f"s={s} t={t}: results lost"
    _E(got, ref, _ebar(a, b) + (K // 1024) * 2.0 ** -149, f"chunked gemm s={s} t={t}")


@pytest.mark.parametrize("K", [256, 2048])
@pytest.mark.parametrize("act", [None, "relu"])
def test_dense_scale_equivariance(ops, act, K):
  B, N = 1024, 128
  x = _rand_away_from_zero((B, K), 95); W = _rand_away_from_zero((K, N), 96); b = _rand_away_from_zero((N,), 97)
  with torch.no_grad():
    base = ops.dense(x, W, b, act)
    for s, t in [(-60, -50), (40, 30), (-100, 90), (100, -20), (-70, -40)]:
      got = ops.dense(_sc(x, s), _sc(W, t), _sc(b, s + t), act)
      _assert_scaled_bits(got, base, s + t, f"dense {act} K={K} s={s} t={t}")


def test_cross_scale_equivariance(ops):
  B, D = 1024, 200
  x0 = _rand_away_from_zero((B, D), 98); x = _rand_away_from_zero((B, D), 99)
  W = _rand_away_from_zero((D, D), 100); b = _rand_away_from_zero((D,), 101)
  with torch.no_grad():
    base = ops.cross(x0, x, W, b, 0.5)
    for s in [-100, -60, 60, 100]:
      _assert_scaled_bits(ops.cross(x0, _sc(x, s), W, _sc(b, s), 0.5), base, s, f"cross s={s}")


def _log_scales(n, lo, hi, seed):
  return torch.exp2(torch.from_numpy(np.random.RandomState(seed).uniform(lo, hi, n)).float().cuda())


@pytest.mark.parametrize("K", [700, 3000])
@pytest.mark.parametrize("ta,tb", [(False, False), (True, True)])
def test_gemm_heterogeneous_magnitudes(ops, ta, tb, K):
  """Rows of A and columns of B at 2^u, u uniform in [-30, 0]: bar (T) cannot see the small rows, bar (E) can."""
  M, N = 320, 192
  ra, cb = _log_scales(M, -30, 0, 1), _log_scales(N, -30, 0, 2)
  A, Bm = _operands(ta, tb, M, N, K, 103)
  A = A * (ra[None, :] if ta else ra[:, None]); Bm = Bm * (cb[:, None] if tb else cb[None, :])
  a, b = _op64(ta, tb, M, N, K, A, Bm)
  _E(_f64(_gemm(ops, ta, tb, M, N, K, A, Bm)), a @ b, _ebar(a, b), f"gemm K={K} ta={ta} tb={tb}")


def test_dense_heterogeneous_magnitudes(ops):
  """Per-row (batch) and per-feature scales of x: each output meets (E) plus 2^-22 of |bias| (the epilogue's add)."""
  B, K, N = 1024, 300, 128
  x = _rand((B, K), 105) * _log_scales(B, -30, 0, 3)[:, None] * _log_scales(K, -30, 0, 4)[None, :]
  W = _rand((K, N), 106, K ** -0.5); b = _rand((N,), 107, 1e-6)
  with torch.no_grad():
    y = _f64(ops.dense(x, W, b, None))
  x64, W64, b64 = _f64(x), _f64(W), _f64(b)
  _E(y, x64 @ W64 + b64, _ebar(x64, W64) + 2.0 ** -22 * np.abs(b64)[None, :], "dense (E)")


def test_cross_heterogeneous_magnitudes(ops):
  """Per-row and per-feature scales of x: out = x0 (x W + b + diag x) + x meets |x0| (E of x W) + 2^-22 of each term."""
  B, D = 1024, 256
  x0 = _rand((B, D), 108, 0.5)
  x = _rand((B, D), 109) * _log_scales(B, -30, 0, 5)[:, None] * _log_scales(D, -30, 0, 6)[None, :]
  W = _rand((D, D), 110, D ** -0.5); b = _rand((D,), 111, 1e-9)
  with torch.no_grad():
    out = _f64(ops.cross(x0, x, W, b, 0.5))
  x0_, x_, W_, b_ = _f64(x0), _f64(x), _f64(W), _f64(b)
  prod = x_ @ W_ + b_ + 0.5 * x_
  tol = np.abs(x0_) * (_ebar(x_, W_) + 2.0 ** -22 * (np.abs(b_) + 0.5 * np.abs(x_))) + 2.0 ** -22 * (np.abs(x0_ * prod) + np.abs(x_))
  _E(out, x0_ * prod + x_, tol, "cross (E)")


def test_gemm_huge_product_of_scales(ops):
  """amax_A * amax_B >= 2^156 (A's largest row at 2^100, B's largest column at 2^60): 2^-(exp_a + exp_b) overflows.  A row
  of zeros and a row of magnitude 1 (which flushes to zero in fp16) must come out finite and meet (E); the one element
  whose float64 value overflows fp32 must be non-finite."""
  M, N, K = 256, 128, 512
  ra = torch.exp2(torch.from_numpy(np.random.RandomState(7).uniform(0, 40, M)).float()).cuda()
  ra[0] = 2.0 ** 100; ra[1] = 0.0; ra[2] = 1.0
  cb = torch.exp2(torch.from_numpy(np.random.RandomState(8).uniform(0, 10, N)).float()).cuda()
  cb[0] = 2.0 ** 60
  A = _rand((M, K), 113) * ra[:, None]; Bm = _rand((K, N), 114) * cb[None, :]
  assert float(A.abs().max()) * float(Bm.abs().max()) >= 2.0 ** 156
  got = _f64(_gemm(ops, False, False, M, N, K, A, Bm))
  a, b = _f64(A), _f64(Bm)
  ref = a @ b
  assert np.isfinite(got[1:3]).all(), "the zero row / the unit row are not finite"
  _E(got, ref, _ebar(a, b), "gemm 2^156")


def _plant(t, i, j, v):
  t = t.clone(); t[i, j] = v; return t


@pytest.mark.parametrize("scale", [2.0 ** -12, 2.0 ** -18, 1.0])
@pytest.mark.parametrize("where,val", [("A", float("inf")), ("B", float("-inf")), ("A", float("nan")), ("B", float("nan"))])
def test_gemm_one_non_finite_input(ops, where, val, scale):
  """One Inf or NaN makes only its own row of C (in A) or column (in B) non-finite; every other element meets (E) -- the
  rescale statistic is the max over the finite entries.  At scale 2^-18 an unscaled operand would lose its lo halves."""
  M, N, K = 256, 256, 1024
  A, Bm = _rand((M, K), 115, scale), _rand((K, N), 116, scale)
  if where == "A":
    A = _plant(A, 37, 500, val)
  else:
    Bm = _plant(Bm, 501, 41, val)
  got = _f64(_gemm(ops, False, False, M, N, K, A, Bm))
  a, b = _f64(A), _f64(Bm)
  ref = a @ b
  bad = np.zeros((M, N), bool)
  if where == "A":
    bad[37, :] = True
  else:
    bad[:, 41] = True
  assert not np.isfinite(got[bad]).any(), "the row / column of the non-finite input is finite"
  _E(got, np.where(bad, 0.0, ref), _ebar(a, b), "gemm (E) off the non-finite row / column", check=~bad)


@pytest.mark.parametrize("val", [float("inf"), float("nan")])
def test_cross_one_non_finite_input(ops, val):
  """A non-finite element of x spoils its own row of out; the other rows meet (E), and out_amax skips it."""
  B, D = 1024, 256
  x0 = _rand((B, D), 117, 0.5); x = _plant(_rand((B, D), 118, 2.0 ** -18), 300, 7, val)
  W = _rand((D, D), 119, D ** -0.5)
  out, prod, amax = _cross_fwd_raw(ops, x0, x, W, None, B, D, D, 0.0)
  got = _f64(out)
  x0_, x_, W_ = _f64(x0), _f64(x), _f64(W)
  assert not np.isfinite(got[300]).any()
  keep = np.ones(B, bool); keep[300] = False
  xk = x_[keep]
  p = xk @ W_
  tol = np.abs(x0_[keep]) * _ebar(xk, W_) + 2.0 ** -22 * (np.abs(x0_[keep] * p) + np.abs(xk))
  _E(got[keep], x0_[keep] * p + xk, tol, "cross (E) off the non-finite row")
  finite = out[torch.isfinite(out)]
  assert int(amax.item()) == int(finite.abs().max().view(torch.int32).item()), "out_amax is not max over the finite |out|"


def test_zero_operands(ops):
  """gemm_tc of a zero operand is +0.0 everywhere; Dense with W = 0 is act(bias); Cross with W = 0, no bias, is x."""
  M, N, K = 300, 200, 1500
  for ta, tb in TRANS:
    A, Bm = _operands(ta, tb, M, N, K, 121)
    for a_, b_ in [(torch.zeros_like(A), Bm), (A, torch.zeros_like(Bm))]:
      assert (_bits(_gemm(ops, ta, tb, M, N, K, a_, b_)) == 0).all()
  B, Kd, Nd = 1024, 300, 128
  x = _rand((B, Kd), 122); b = _rand((Nd,), 123)
  W0 = torch.zeros((Kd, Nd), device="cuda")
  with torch.no_grad():
    assert torch.equal(_bits(ops.dense(x, W0, b, None)), _bits(b.expand(B, Nd)))
    assert torch.equal(_bits(ops.dense(x, W0, b, "relu")), _bits(torch.where(b > 0, b, torch.zeros_like(b)).expand(B, Nd)))
    y = ops.dense(x, W0, b, "sigmoid")
    assert torch.equal(_bits(ops.attached_logits(y)), _bits(b.expand(B, Nd)))
    x0 = _rand((B, 256), 124); xc = _rand((B, 256), 125)
    assert torch.equal(_bits(ops.cross(x0, xc, torch.zeros((256, 256), device="cuda"), None, 0.0)), _bits(xc))


# ------------------------------------------------------------------------------------------------
# Determinism
# ------------------------------------------------------------------------------------------------
def test_every_mode_is_deterministic(ops):
  def same(f, what):
    assert torch.equal(_bits(f()), _bits(f())), what

  for K in (512, 3000):                                                     # PLAIN, chunked PLAIN
    A, Bm = _operands(False, True, 700, 300, K, 131)
    same(lambda: _gemm(ops, False, True, 700, 300, K, A, Bm), f"gemm K={K}")
  with torch.no_grad():
    for K in (256, 2000):                                                   # DENSE x 3 activations, unchunked and chunked
      x = _rand((1024, K), 132); W = _rand((K, 128), 133, K ** -0.5); b = _rand((128,), 134)
      for act in (None, "relu", "sigmoid"):
        same(lambda: ops.dense(x, W, b, act), f"dense K={K} {act}")
        if act == "sigmoid":
          same(lambda: ops.attached_logits(ops.dense(x, W, b, act)), f"dense K={K} logits")
  for B, D in [(1100, 300), (1024, 1100)]:                                  # CROSS with out_amax, DX; single and chunked
    x0, x, g = _rand((B, D), 135), _rand((B, D), 136), _rand((B, D), 137)
    W, b = _rand((D, D), 138, D ** -0.5), _rand((D,), 139)
    runs = [_cross_fwd_raw(ops, x0, x, W, b, B, D, D, 0.5) for _ in range(2)]
    for u, v in zip(*runs):
      assert torch.equal(_bits(u), _bits(v)), f"cross forward D={D}"
    grads = [_cross_bwd_raw(ops, x0, x, W, runs[0][1], g, B, D, D, 0.5) for _ in range(2)]
    for u, v in zip(*grads):
      assert torch.equal(_bits(u), _bits(v)), f"cross backward D={D}"
