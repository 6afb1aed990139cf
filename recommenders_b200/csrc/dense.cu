// dense.cu -- K6: the Dense layer of the ranking MLPs (tf.keras.layers.Dense in layers/blocks.py:24-61 and
// experimental/models/ranking.py:27-257):  y = act(x . W + bias),  W [in, out] as Keras stores it.
//   tensor cores (B >= 1024, K >= 64, N >= 64): split-fp16 wgmma GEMM (split_gemm.cu) with a DENSE epilogue;
//   otherwise exact CUDA-core kernels whose outputs are the canonical sequential fmaf chain + bias + activation
//   (a warp per row for narrow layers, N <= 16, e.g. the Dense(1) logit layer; the exact SGEMM above that).
//   bwd: dz = dy * act'(y) + dlogits (from the saved output) ; db = colsum(dz) (two-level fixed-order float64 reduction) ;
//        dx = dz . W^T ; dW = x^T . dz (batch cut into chunks, partials summed in fixed order).  No float atomics.
#include "sgemm.cuh"
#include "split_gemm.cuh"
#include "dense.cuh"

namespace tfrs {

constexpr int DENSE_NARROW_N = 16;     // widest layer that runs the warp-per-row kernel
constexpr int DENSE_COL_SPLITS = 64;   // row splits of the bias-gradient column sum

static bool dense_tc(long long B, int K, int N) { return B >= 1024 && K >= 64 && N >= 64 && B < (1ll << 31); }

struct EpiDense {
  const float* bias; int act; long long ld; float* y; float* logits;
  __device__ __forceinline__ void operator()(int m, int n, float acc, int) const {
    const long long o = (long long)m * ld + n;
    const float z = bias ? acc + bias[n] : acc;
    if (logits) logits[o] = z;
    y[o] = dense_act(act, z);
  }
};

// one warp per row: lane j < N owns output j; x is read coalesced, 32 k at a time, and broadcast by shuffle, so every output
// is the sequential chain acc = fmaf(x[k], W[k, j], acc), k ascending from +0.0f
__global__ void __launch_bounds__(256)
dense_narrow_fwd_kernel(const float* __restrict__ x, const float* __restrict__ W, const float* __restrict__ bias, long long B, int K,
                        int N, int act, float* __restrict__ y, float* __restrict__ logits) {
  const int lane = threadIdx.x & 31;
  const long long row = ((long long)blockIdx.x * 256 + threadIdx.x) >> 5;
  if (row >= B) return;
  const float* xr = x + row * K;
  float acc = 0.f;
  for (int k0 = 0; k0 < K; k0 += 32) {
    const float xv = k0 + lane < K ? __ldg(xr + k0 + lane) : 0.f;
    const int kn = min(32, K - k0);
    for (int kk = 0; kk < kn; ++kk) {
      const float a = __shfl_sync(0xffffffffu, xv, kk);
      if (lane < N) acc = fmaf(a, __ldg(W + (long long)(k0 + kk) * N + lane), acc);
    }
  }
  if (lane < N) {
    const float z = bias ? acc + bias[lane] : acc;
    if (logits) logits[row * N + lane] = z;
    y[row * N + lane] = dense_act(act, z);
  }
}

// dz = dy * act'(y) + dlogits   (either input may be absent)
__global__ void __launch_bounds__(256)
dense_dz_kernel(const float* __restrict__ y, const float* __restrict__ dy, const float* __restrict__ dl, long long total, int act,
                float* __restrict__ dz) {
  for (long long e = (long long)blockIdx.x * 256 + threadIdx.x; e < total; e += (long long)gridDim.x * 256) {
    float v = dy ? dense_act_grad(act, y[e], dy[e]) : dl[e];
    if (dy && dl) v += dl[e];
    dz[e] = v;
  }
}

// partial[z][n] = sum over the rows of split z (ascending), in float64: a narrow layer's bias gradient is one long sum whose
// terms largely cancel, so fp32 partial sums would leave an error of the order of the result
__global__ void __launch_bounds__(256)
dense_colsum_partial(const float* __restrict__ dz, long long B, int N, long long rows_per_split, double* __restrict__ partial) {
  const int n = blockIdx.x * 256 + threadIdx.x;
  if (n >= N) return;
  const long long r0 = (long long)blockIdx.y * rows_per_split;
  const long long r1 = r0 + rows_per_split < B ? r0 + rows_per_split : B;
  double a = 0.0;
  for (long long r = r0; r < r1; ++r) a += (double)dz[r * N + n];
  partial[(long long)blockIdx.y * N + n] = a;
}

__global__ void __launch_bounds__(256)
dense_colsum_reduce(const double* __restrict__ partial, int N, int splits, float* __restrict__ out) {
  const int n = blockIdx.x * 256 + threadIdx.x;
  if (n >= N) return;
  double a = partial[n];
  for (int z = 1; z < splits; ++z) a += partial[(long long)z * N + n];
  out[n] = (float)a;
}

static size_t dense_bwd_gemm_ws(long long B, int K, int N) {
  if (dense_tc(B, K, N)) {
    const size_t a = tc::gemm_tc_workspace(B, K, N), b = tc::gemm_tc_workspace(K, N, B);
    return a > b ? a : b;
  }
  return (size_t)sgemm_batch_splits(B) * K * N * 4;
}

}  // namespace tfrs
using namespace tfrs;

extern "C" int tfrs_dense_uses_tc(int64_t B, int K, int N) { return dense_tc(B, K, N) ? 1 : 0; }

extern "C" size_t tfrs_dense_fwd_workspace_bytes(int64_t B, int K, int N) {
  return dense_tc(B, K, N) ? tc::gemm_tc_workspace(B, N, K) : 0;
}

extern "C" int tfrs_dense_fwd_f32(const float* x, const float* W, const float* bias, int64_t B, int K, int N, int activation, float* y,
                                  float* logits, void* ws, size_t ws_bytes, void* stream) {
  TFRS_CHECK_ARG(x && W && y, "dense_fwd: NULL pointer");
  TFRS_CHECK_ARG(B >= 0 && K > 0 && N > 0 && B < (1ll << 31), "dense_fwd: bad shape B=%lld K=%d N=%d", (long long)B, K, N);
  TFRS_CHECK_ARG(activation >= TFRS_ACT_LINEAR && activation <= TFRS_ACT_SIGMOID, "dense_fwd: unknown activation %d", activation);
  if (B == 0) return TFRS_OK;
  cudaStream_t st = (cudaStream_t)stream;
  float* lg = activation == TFRS_ACT_SIGMOID ? logits : nullptr;
  if (dense_tc(B, K, N)) {   // image row of the B operand = output n, reduction index k: W[k*N + n]
    const tc::GemmEpilogue ep{tc::GEMM_EPI_DENSE, nullptr, 0, nullptr, 0, bias, 0.f, lg, activation};
    return tc::gemm_tc(tc::GemmOperand{x, K, false}, tc::GemmOperand{W, N, true}, B, N, K, ep, y, N, ws, ws_bytes, st);
  }
  if (N <= DENSE_NARROW_N) {
    dense_narrow_fwd_kernel<<<(unsigned)ceil_div(B * 32, 256), 256, 0, st>>>(x, W, bias, B, K, N, activation, y, lg);
    TFRS_LAUNCH_CHECK();
    return TFRS_OK;
  }
  return launch_sgemm<false, false>(x, K, W, N, (int)B, N, K, 1, EpiDense{bias, activation, N, y, lg}, st);
}

extern "C" size_t tfrs_dense_bwd_workspace_bytes(int64_t B, int K, int N) {
  if (B <= 0 || K <= 0 || N <= 0) return 256;
  return align_up((size_t)B * N * 4, 1024) + align_up((size_t)DENSE_COL_SPLITS * N * 8, 1024) + dense_bwd_gemm_ws(B, K, N);
}

extern "C" int tfrs_dense_bwd_f32(const float* x, const float* W, const float* y, const float* dy, const float* dlogits, int64_t B,
                                  int K, int N, int activation, float* dx, float* dW, float* dbias, void* ws, size_t ws_bytes,
                                  void* stream) {
  TFRS_CHECK_ARG(x && W && y && (dy || dlogits), "dense_bwd: NULL pointer");
  TFRS_CHECK_ARG(B > 0 && K > 0 && N > 0 && B < (1ll << 31), "dense_bwd: bad shape B=%lld K=%d N=%d", (long long)B, K, N);
  TFRS_CHECK_ARG(activation >= TFRS_ACT_LINEAR && activation <= TFRS_ACT_SIGMOID, "dense_bwd: unknown activation %d", activation);
  if (!ws || ws_bytes < tfrs_dense_bwd_workspace_bytes(B, K, N)) { set_error("dense_bwd: workspace too small"); return TFRS_ERR_WORKSPACE_TOO_SMALL; }
  TFRS_CHECK_ARG((reinterpret_cast<uintptr_t>(ws) & 15) == 0, "dense_bwd: workspace must be 16-byte aligned");
  cudaStream_t st = (cudaStream_t)stream;
  unsigned char* w = (unsigned char*)ws;
  float* dz = (float*)w; w += align_up((size_t)B * N * 4, 1024);
  double* colpart = (double*)w; w += align_up((size_t)DENSE_COL_SPLITS * N * 8, 1024);
  const size_t gws = ws_bytes - (size_t)(w - (unsigned char*)ws);
  const long long total = (long long)B * N;
  dense_dz_kernel<<<elementwise_grid(total), 256, 0, st>>>(y, dy, dlogits, total, activation, dz);
  TFRS_LAUNCH_CHECK();
  int rc;
  if (dense_tc(B, K, N)) {
    const tc::GemmEpilogue plain{tc::GEMM_EPI_PLAIN, nullptr, 0, nullptr, 0, nullptr, 0.f, nullptr, 0};
    if (dx) {   // dx[b, i] = sum_o dz[b, o] W[i, o]
      rc = tc::gemm_tc(tc::GemmOperand{dz, N, false}, tc::GemmOperand{W, N, false}, B, K, N, plain, dx, K, w, gws, st);
      if (rc) return rc;
    }
    if (dW) {   // dW[i, o] = sum_b x[b, i] dz[b, o]
      rc = tc::gemm_tc(tc::GemmOperand{x, K, true}, tc::GemmOperand{dz, N, true}, K, N, B, plain, dW, N, w, gws, st);
      if (rc) return rc;
    }
  } else {
    if (dx) {
      rc = launch_sgemm<false, true>(dz, N, W, N, (int)B, K, N, 1, EpiStore{dx, K}, st);
      if (rc) return rc;
    }
    if (dW) {
      rc = launch_sgemm_split_k<true, false>(x, K, dz, N, K, N, (int)B, sgemm_batch_splits(B), (float*)w, dW, st);
      if (rc) return rc;
    }
  }
  if (dbias) {
    const long long rps = ceil_div(B, DENSE_COL_SPLITS);
    const int used = (int)ceil_div(B, rps);
    dense_colsum_partial<<<dim3((unsigned)ceil_div(N, 256), (unsigned)used), 256, 0, st>>>(dz, B, N, rps, colpart);
    TFRS_LAUNCH_CHECK();
    dense_colsum_reduce<<<(unsigned)ceil_div(N, 256), 256, 0, st>>>(colpart, N, used, dbias);
    TFRS_LAUNCH_CHECK();
  }
  return TFRS_OK;
}
