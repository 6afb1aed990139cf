// cross.cu -- K5/K5b: DCN-v2 cross layer, full-rank (layers/feature_interaction/dcn.py:176-186) and low-rank.
//   fwd: out = x0 * (x . W + bias + diag_scale * x) + x     W is [in,out] (Keras Dense, dcn.py:121-130)
//        one GEMM whose epilogue applies bias / diag / x0 / residual, so the [B,D] product never makes a separate HBM
//        round trip (the reference runs MatMul, BiasAdd, Mul, Add): the exact SGEMM (sgemm.cuh) for small shapes, the
//        split-fp16 tensor-core GEMM (split_gemm.cu) otherwise.
//   bwd: gp = g*x0 ; dx0 = g*prod ; dx = gp . W^T + diag*gp + g ; dW = x^T . gp (deterministic split-K) ;
//        dbias = colsum(gp) (two-level fixed-order reduction).
#include "sgemm.cuh"
#include "split_gemm.cuh"

namespace tfrs {

struct EpiCrossFwd {
  const float* x0; const float* x; const float* bias; float diag; long long ld; float* out; float* prod;
  __device__ __forceinline__ void operator()(int m, int n, float acc, int) const {
    long long o = (long long)m * ld + n;
    float xv = x[o];
    float p = acc;
    if (bias) p += bias[n];
    if (diag != 0.f) p += diag * xv;
    if (prod) prod[o] = p;
    out[o] = x0[o] * p + xv;
  }
};

struct EpiCrossDx {
  const float* gp; long long ldgp; const float* g; long long ld; float diag; float* dx;
  __device__ __forceinline__ void operator()(int m, int n, float acc, int) const {
    float v = acc + g[(long long)m * ld + n];
    if (diag != 0.f) v += diag * gp[(long long)m * ldgp + n];
    dx[(long long)m * ld + n] = v;
  }
};

// gp = g * x0 (dense [B,D]); dx0 = g * prod; optionally max |gp| over the finite elements (bits of a non-negative float,
// one atomic per CTA) for the tensor-core path's power-of-two rescale.
__global__ void __launch_bounds__(256)
cross_bwd_elem(const float* __restrict__ x0, const float* __restrict__ prod, const float* __restrict__ g,
               long long B, int D, long long ld, float* __restrict__ gp, float* __restrict__ dx0,
               unsigned int* __restrict__ gp_amax_bits) {
  const long long total = B * D;
  float amax = 0.f;
  for (long long e = (long long)blockIdx.x * 256 + threadIdx.x; e < total; e += (long long)gridDim.x * 256) {
    long long m = e / D; int n = (int)(e - m * D);
    long long o = m * ld + n;
    float gv = g[o];
    const float v = gv * x0[o];
    gp[e] = v;
    amax = fmaxf(amax, finite_abs(v));
    if (dx0) dx0[o] = gv * prod[o];
  }
  if (gp_amax_bits) {
    __shared__ float red[8];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = amax;
    __syncthreads();
    if (threadIdx.x == 0) {
#pragma unroll
      for (int i = 1; i < 8; ++i) amax = fmaxf(amax, red[i]);
      if (amax > 0.f) atomicMax(gp_amax_bits, __float_as_uint(amax));
    }
  }
}

// partial[z][n] = sum over rows of split z (fixed order)
__global__ void __launch_bounds__(256)
cross_colsum_partial(const float* __restrict__ gp, long long B, int D, long long rows_per_split, float* __restrict__ partial) {
  int n = blockIdx.x * 256 + threadIdx.x;
  if (n >= D) return;
  long long r0 = (long long)blockIdx.y * rows_per_split;
  long long r1 = r0 + rows_per_split < B ? r0 + rows_per_split : B;
  float a = 0.f;
  long long r = r0;
  for (; r + 8 <= r1; r += 8) {  // 8 independent loads in flight, summed in row order (same result as the plain loop)
    float v[8];
#pragma unroll
    for (int u = 0; u < 8; ++u) v[u] = gp[(r + u) * D + n];
#pragma unroll
    for (int u = 0; u < 8; ++u) a += v[u];
  }
  for (; r < r1; ++r) a += gp[r * D + n];
  partial[(long long)blockIdx.y * D + n] = a;
}

constexpr int CROSS_COL_SPLITS = 64;

// dbias = colsum(gp): row-split partials, then their fixed-order sum
static int cross_colsum(const float* gp, long long B, int D, float* colpart, float* dbias, cudaStream_t st) {
  const long long rps = ceil_div(B, CROSS_COL_SPLITS);
  const int used = (int)ceil_div(B, rps);
  cross_colsum_partial<<<dim3((unsigned)ceil_div(D, 256), (unsigned)used), 256, 0, st>>>(gp, B, D, rps, colpart);
  TFRS_LAUNCH_CHECK();
  return reduce_parts(colpart, 1, D, used, dbias, D, st);
}

}  // namespace tfrs
using namespace tfrs;

extern "C" int tfrs_cross_fwd_f32(const float* x0, const float* x, const float* W, const float* bias, int64_t B,
                                  int D, int64_t ld, float diag_scale, float* out, float* prod, void* stream) {
  TFRS_CHECK_ARG(x0 && x && W && out, "cross_fwd: NULL pointer");
  TFRS_CHECK_ARG(B >= 0 && D > 0 && ld >= D, "cross_fwd: bad shape B=%lld D=%d ld=%lld", (long long)B, D, (long long)ld);
  TFRS_CHECK_ARG(diag_scale >= 0.f, "`diag_scale` should be non-negative. Got `diag_scale` = %g", diag_scale);
  TFRS_CHECK_ARG(B < (1ll << 31), "cross_fwd: B too large");
  if (B == 0) return TFRS_OK;
  EpiCrossFwd epi{x0, x, bias, diag_scale, ld, out, prod};
  return launch_sgemm<false, false>(x, ld, W, D, (int)B, D, D, 1, epi, (cudaStream_t)stream);
}

extern "C" size_t tfrs_cross_bwd_workspace_bytes(int64_t B, int D) {
  if (B <= 0 || D <= 0) return 256;
  return align_up((size_t)B * D * 4, 256) + align_up((size_t)sgemm_batch_splits(B) * D * D * 4, 256) +
         align_up((size_t)CROSS_COL_SPLITS * D * 4, 256);
}

extern "C" int tfrs_cross_bwd_f32(const float* x0, const float* x, const float* W, const float* prod,
                                  const float* dout, int64_t B, int D, int64_t ld, float diag_scale, float* dx0,
                                  float* dx, float* dW, float* dbias, void* ws, size_t ws_bytes, void* stream) {
  TFRS_CHECK_ARG(x0 && x && W && dout, "cross_bwd: NULL pointer");
  TFRS_CHECK_ARG(B > 0 && D > 0 && ld >= D && B < (1ll << 31), "cross_bwd: bad shape");
  TFRS_CHECK_ARG(!dx0 || prod, "cross_bwd: dx0 needs the saved `prod`");
  if (!ws || ws_bytes < tfrs_cross_bwd_workspace_bytes(B, D)) { set_error("cross_bwd: workspace too small"); return TFRS_ERR_WORKSPACE_TOO_SMALL; }
  cudaStream_t st = (cudaStream_t)stream;
  unsigned char* w = (unsigned char*)ws;
  float* gp = (float*)w; w += align_up((size_t)B * D * 4, 256);
  const int Z = sgemm_batch_splits(B);
  float* part = (float*)w; w += align_up((size_t)Z * D * D * 4, 256);
  float* colpart = (float*)w;

  cross_bwd_elem<<<elementwise_grid((long long)B * D), 256, 0, st>>>(x0, prod, dout, B, D, ld, gp, dx0, nullptr);
  TFRS_LAUNCH_CHECK();
  int rc;
  if (dx) {
    rc = launch_sgemm<false, true>(gp, D, W, D, (int)B, D, D, 1, EpiCrossDx{gp, D, dout, ld, diag_scale, dx}, st);
    if (rc) return rc;
  }
  if (dW) {
    rc = launch_sgemm_split_k<true, false>(x, ld, gp, D, D, D, (int)B, Z, part, dW, st);
    if (rc) return rc;
  }
  return dbias ? cross_colsum(gp, B, D, colpart, dbias, st) : TFRS_OK;
}

// ---- K5 / K5b on the tensor cores: one split-fp16 GEMM forward, two backward; same contract and outputs as the exact path
extern "C" size_t tfrs_cross_tc_workspace_bytes(int64_t B, int D) {
  return tc::gemm_tc_workspace(B, D, D);
}

extern "C" int tfrs_cross_tc_fwd_f32(const float* x0, const float* x, const float* W, const float* bias, int64_t B, int D, int64_t ld,
                                     float diag_scale, float* out, float* prod, const unsigned int* x_amax_bits,
                                     unsigned int* out_amax_bits, void* ws, size_t ws_bytes, void* stream) {
  TFRS_CHECK_ARG(x0 && x && W && out, "cross_tc_fwd: NULL pointer");
  TFRS_CHECK_ARG(B > 0 && D > 0 && ld >= D, "cross_tc_fwd: bad shape");
  TFRS_CHECK_ARG(diag_scale >= 0.f, "`diag_scale` should be non-negative. Got `diag_scale` = %g", diag_scale);
  // image row of the B operand = output column n, reduction index k: W[k*D + n]
  return tc::gemm_tc(tc::GemmOperand{x, ld, false, x_amax_bits}, tc::GemmOperand{W, D, true}, B, D, D,
                     tc::GemmEpilogue{tc::GEMM_EPI_CROSS, x0, ld, x, ld, bias, diag_scale, prod, 0, out_amax_bits}, out, ld, ws,
                     ws_bytes, (cudaStream_t)stream);
}

// gp | colsum partials | max |gp| | one GEMM workspace shared by the dx and dW calls
extern "C" size_t tfrs_cross_tc_bwd_workspace_bytes(int64_t B, int D) {
  if (B <= 0 || D <= 0) return 0;
  const size_t dx_ws = tc::gemm_tc_workspace(B, D, D), dw_ws = tc::gemm_tc_workspace(D, D, B);
  return align_up((size_t)B * D * 4, 1024) + align_up((size_t)CROSS_COL_SPLITS * D * 4, 1024) + 1024 + (dx_ws > dw_ws ? dx_ws : dw_ws);
}

extern "C" int tfrs_cross_tc_bwd_f32(const float* x0, const float* x, const float* W, const float* prod,
                                     const float* dout, int64_t B, int D, int64_t ld, float diag_scale, float* dx0,
                                     float* dx, float* dW, float* dbias, void* ws, size_t ws_bytes, void* stream) {
  TFRS_CHECK_ARG(x0 && x && W && dout, "cross_tc_bwd: NULL pointer");
  TFRS_CHECK_ARG(B > 0 && D > 0 && ld >= D && B < (1ll << 31), "cross_tc_bwd: bad shape");
  TFRS_CHECK_ARG(!dx0 || prod, "cross_tc_bwd: dx0 needs the saved `prod`");
  if (!ws || ws_bytes < tfrs_cross_tc_bwd_workspace_bytes(B, D)) { set_error("cross_tc_bwd: workspace too small"); return TFRS_ERR_WORKSPACE_TOO_SMALL; }
  TFRS_CHECK_ARG((reinterpret_cast<uintptr_t>(ws) & 15) == 0, "cross_tc_bwd: workspace must be 16-byte aligned");
  cudaStream_t st = (cudaStream_t)stream;
  unsigned char* w = (unsigned char*)ws;
  float* gp = (float*)w; w += align_up((size_t)B * D * 4, 1024);
  float* colpart = (float*)w; w += align_up((size_t)CROSS_COL_SPLITS * D * 4, 1024);
  unsigned int* gp_amax = (unsigned int*)w; w += 1024;
  const size_t gws = ws_bytes - (size_t)(w - (unsigned char*)ws);
  // max |gp| comes out of the element-wise pass: the two GEMMs skip their statistics pass over gp
  TFRS_CUDA(cudaMemsetAsync(gp_amax, 0, sizeof(unsigned int), st));
  cross_bwd_elem<<<elementwise_grid((long long)B * D), 256, 0, st>>>(x0, prod, dout, B, D, ld, gp, dx0, gp_amax);
  TFRS_LAUNCH_CHECK();
  int rc;
  if (dx) {   // dx[b, i] = sum_o gp[b, o] W[i, o] + diag gp[b, i] + g[b, i]
    rc = tc::gemm_tc(tc::GemmOperand{gp, D, false, gp_amax}, tc::GemmOperand{W, D, false}, B, D, D,
                     tc::GemmEpilogue{tc::GEMM_EPI_DX, gp, D, dout, ld, nullptr, diag_scale, nullptr}, dx, ld, w, gws, st);
    if (rc) return rc;
  }
  if (dW) {   // dW[i, o] = sum_b x[b, i] gp[b, o]
    rc = tc::gemm_tc(tc::GemmOperand{x, ld, true}, tc::GemmOperand{gp, D, true, gp_amax}, D, D, B,
                     tc::GemmEpilogue{tc::GEMM_EPI_PLAIN, nullptr, 0, nullptr, 0, nullptr, 0.f, nullptr}, dW, D, w, gws, st);
    if (rc) return rc;
  }
  return dbias ? cross_colsum(gp, B, D, colpart, dbias, st) : TFRS_OK;
}

// ---- general tensor-core GEMM (the low-rank Cross projections; ops.matmul on large shapes) --------------------------------
//   C[M,N] = opA(A) . opB(B),  opA(m,k) = transA ? A[k*lda + m] : A[m*lda + k],  opB(k,n) = transB ? B[n*ldb + k] : B[k*ldb + n]
extern "C" size_t tfrs_gemm_tc_workspace_bytes(int64_t M, int64_t N, int64_t K) { return tc::gemm_tc_workspace(M, N, K); }

extern "C" int tfrs_gemm_tc_f32(int transA, int transB, int64_t M, int64_t N, int64_t K, const float* A, int64_t lda, const float* B,
                                int64_t ldb, float* C, int64_t ldc, void* ws, size_t ws_bytes, void* stream) {
  TFRS_CHECK_ARG(A && B && C, "gemm_tc: NULL pointer");
  TFRS_CHECK_ARG(M > 0 && N > 0 && K > 0 && ldc >= N, "gemm_tc: bad shape");
  TFRS_CHECK_ARG(lda >= (transA ? M : K) && ldb >= (transB ? K : N), "gemm_tc: lda=%lld / ldb=%lld below the row length",
                 (long long)lda, (long long)ldb);
  const tc::GemmOperand a{A, lda, transA != 0};
  const tc::GemmOperand b{B, ldb, transB == 0};   // image rows = n, reduction index k: B[k*ldb + n] is the "transposed" read
  const tc::GemmEpilogue ep{tc::GEMM_EPI_PLAIN, nullptr, 0, nullptr, 0, nullptr, 0.f, nullptr};
  return tc::gemm_tc(a, b, M, N, K, ep, C, ldc, ws, ws_bytes, (cudaStream_t)stream);
}

// ---- low-rank Cross on the tensor cores (dcn.py:131-148,178-179; multi_layer_dcn.py:146-148) -------------------------------
//   t = x . U   [B,p]        (U [D,p]: Dense(projection_dim, use_bias=False))
//   out = x0 * (t . V + bias + diag * x) + x      (V [p,D]: Dense(D)) -- the cross formula is the second GEMM's epilogue
namespace tfrs {
static size_t lr_gemm_ws(long long B, int D, int p) {
  size_t a = tc::gemm_tc_workspace(B, p, D), b = tc::gemm_tc_workspace(B, D, p);
  size_t c = tc::gemm_tc_workspace(p, D, B), d = tc::gemm_tc_workspace(D, p, B);
  size_t m = a > b ? a : b; m = m > c ? m : c; return m > d ? m : d;
}
}  // namespace tfrs

extern "C" size_t tfrs_cross_lowrank_tc_workspace_bytes(int64_t B, int D, int p) {
  if (B <= 0 || D <= 0 || p <= 0) return 0;
  const size_t a = tc::gemm_tc_workspace(B, p, D), b = tc::gemm_tc_workspace(B, D, p);
  return a > b ? a : b;
}

extern "C" int tfrs_cross_lowrank_tc_fwd_f32(const float* x0, const float* x, const float* U, const float* V, const float* bias,
                                             int64_t B, int D, int p, int64_t ld, float diag_scale, float* out, float* prod,
                                             float* t, void* ws, size_t ws_bytes, void* stream) {
  TFRS_CHECK_ARG(x0 && x && U && V && out && t, "cross_lowrank_tc_fwd: NULL pointer");
  TFRS_CHECK_ARG(B > 0 && D > 0 && p > 0 && ld >= D, "cross_lowrank_tc_fwd: bad shape");
  TFRS_CHECK_ARG(diag_scale >= 0.f, "`diag_scale` should be non-negative. Got `diag_scale` = %g", diag_scale);
  if (D > 1024 || p > 1024) { set_error("cross_lowrank_tc_fwd: needs D, projection_dim <= 1024"); return TFRS_ERR_UNSUPPORTED; }
  cudaStream_t st = (cudaStream_t)stream;
  // t = x . U : image rows of B' = the p outputs, element (n, k) = U[k*p + n]
  int rc = tc::gemm_tc(tc::GemmOperand{x, ld, false}, tc::GemmOperand{U, p, true}, B, p, D,
                       tc::GemmEpilogue{tc::GEMM_EPI_PLAIN, nullptr, 0, nullptr, 0, nullptr, 0.f, nullptr}, t, p, ws, ws_bytes, st);
  if (rc) return rc;
  // out = x0 * (t . V + bias + diag x) + x : element (n, k) = V[k*D + n]
  return tc::gemm_tc(tc::GemmOperand{t, p, false}, tc::GemmOperand{V, D, true}, B, D, p,
                     tc::GemmEpilogue{tc::GEMM_EPI_CROSS, x0, ld, x, ld, bias, diag_scale, prod}, out, ld, ws, ws_bytes, st);
}

// backward:  gp = g * x0 ; dx0 = g * prod ; dt = gp . V^T ; dV = t^T . gp ; dU = x^T . dt ; dx = dt . U^T + diag * gp + g ;
//            dbias = colsum(gp).  All four GEMMs on the tensor cores (the two batch-long reductions chunked, partials summed
//            in fixed order): deterministic.
extern "C" size_t tfrs_cross_lowrank_tc_bwd_workspace_bytes(int64_t B, int D, int p) {
  if (B <= 0 || D <= 0 || p <= 0) return 0;
  return align_up((size_t)B * D * 4, 1024) + align_up((size_t)B * p * 4, 1024) + align_up((size_t)CROSS_COL_SPLITS * D * 4, 1024) +
         lr_gemm_ws(B, D, p);
}

extern "C" int tfrs_cross_lowrank_tc_bwd_f32(const float* x0, const float* x, const float* U, const float* V, const float* t,
                                             const float* prod, const float* dout, int64_t B, int D, int p, int64_t ld,
                                             float diag_scale, float* dx0, float* dx, float* dU, float* dV, float* dbias, void* ws,
                                             size_t ws_bytes, void* stream) {
  TFRS_CHECK_ARG(x0 && x && U && V && t && dout, "cross_lowrank_tc_bwd: NULL pointer");
  TFRS_CHECK_ARG(B > 0 && D > 0 && p > 0 && ld >= D && B < (1ll << 31), "cross_lowrank_tc_bwd: bad shape");
  TFRS_CHECK_ARG(!dx0 || prod, "cross_lowrank_tc_bwd: dx0 needs the saved `prod`");
  if (D > 1024 || p > 1024) { set_error("cross_lowrank_tc_bwd: needs D, projection_dim <= 1024"); return TFRS_ERR_UNSUPPORTED; }
  if (!ws || ws_bytes < tfrs_cross_lowrank_tc_bwd_workspace_bytes(B, D, p)) { set_error("cross_lowrank_tc_bwd: workspace too small"); return TFRS_ERR_WORKSPACE_TOO_SMALL; }
  TFRS_CHECK_ARG((reinterpret_cast<uintptr_t>(ws) & 15) == 0, "cross_lowrank_tc_bwd: workspace must be 16-byte aligned");
  cudaStream_t st = (cudaStream_t)stream;
  unsigned char* w = (unsigned char*)ws;
  float* gp = (float*)w; w += align_up((size_t)B * D * 4, 1024);
  float* dt = (float*)w; w += align_up((size_t)B * p * 4, 1024);
  float* colpart = (float*)w; w += align_up((size_t)CROSS_COL_SPLITS * D * 4, 1024);
  const size_t gws = ws_bytes - (size_t)(w - (unsigned char*)ws);
  cross_bwd_elem<<<elementwise_grid((long long)B * D), 256, 0, st>>>(x0, prod, dout, B, D, ld, gp, dx0, nullptr);
  TFRS_LAUNCH_CHECK();
  const tc::GemmEpilogue plain{tc::GEMM_EPI_PLAIN, nullptr, 0, nullptr, 0, nullptr, 0.f, nullptr};
  int rc;
  if (dx || dU) {   // dt[b, j] = sum_o gp[b, o] V[j, o]
    rc = tc::gemm_tc(tc::GemmOperand{gp, D, false}, tc::GemmOperand{V, D, false}, B, p, D, plain, dt, p, w, gws, st);
    if (rc) return rc;
  }
  if (dV) {         // dV[j, o] = sum_b t[b, j] gp[b, o]
    rc = tc::gemm_tc(tc::GemmOperand{t, p, true}, tc::GemmOperand{gp, D, true}, p, D, B, plain, dV, D, w, gws, st);
    if (rc) return rc;
  }
  if (dU) {         // dU[i, j] = sum_b x[b, i] dt[b, j]
    rc = tc::gemm_tc(tc::GemmOperand{x, ld, true}, tc::GemmOperand{dt, p, true}, D, p, B, plain, dU, p, w, gws, st);
    if (rc) return rc;
  }
  if (dx) {         // dx[b, i] = sum_j dt[b, j] U[i, j] + diag gp[b, i] + g[b, i]
    rc = tc::gemm_tc(tc::GemmOperand{dt, p, false}, tc::GemmOperand{U, p, false}, B, D, p,
                     tc::GemmEpilogue{tc::GEMM_EPI_DX, gp, D, dout, ld, nullptr, diag_scale, nullptr}, dx, ld, w, gws, st);
    if (rc) return rc;
  }
  return dbias ? cross_colsum(gp, B, D, colpart, dbias, st) : TFRS_OK;
}
