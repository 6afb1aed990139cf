// sgemm.cuh -- exact fp32 CUDA-core GEMM with a functor epilogue.
//
//   C[m,n] = sum_{k=k_begin}^{k_end-1} opA(m,k) * opB(k,n)
//   opA(m,k) = TA ? A[k*lda + m] : A[m*lda + k]      opB(k,n) = TB ? B[n*ldb + k] : B[k*ldb + n]
//
// Every output element is accumulated by ONE thread as the sequential chain
//   acc = fmaf(a_k, b_k, acc),  k ascending, acc starting at +0.0f
// which is the canonical arithmetic of this repo (oracle/tfrs_oracle.c dot_chain): results are
// bit-identical to the oracle, so this kernel is the correctness anchor for the tensor-core paths.
// The K tail is never padded with zero products (keeps -0.0f exact).
#pragma once
#include "common.cuh"

namespace tfrs {

constexpr int SG_BM = 128, SG_BN = 128, SG_BK = 16, SG_THREADS = 256;

template <bool TA, bool TB, int BN, class Epi>
__global__ void __launch_bounds__(SG_THREADS)
sgemm_kernel(const float* __restrict__ A, long long lda, const float* __restrict__ B, long long ldb,
             int M, int N, int K, int k_per_split, bool vecA, bool vecB, Epi epi) {
  __shared__ __align__(16) float As[SG_BK][SG_BM + 4];
  constexpr int TN = BN / 16;  // columns per thread (8 for BN=128, 4 for the skinny BN=64 variant)
  __shared__ __align__(16) float Bs[SG_BK][BN + 4];

  const int tid = threadIdx.x;
  const int m0 = blockIdx.y * SG_BM, n0 = blockIdx.x * BN;
  const int k_begin = blockIdx.z * k_per_split;
  const int k_end = min(K, k_begin + k_per_split);
  const int tx = tid % 16, ty = tid / 16;

  float acc[8][TN];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < TN; ++j) acc[i][j] = 0.0f;

  for (int k0 = k_begin; k0 < k_end; k0 += SG_BK) {
    const int kmax = min(SG_BK, k_end - k0);
    // ---- load A tile -> As[k][m]
    if (!TA) {
      if (vecA) {  // float4 along k; requires lda % 4 == 0, 16B-aligned base, k_begin % 4 == 0
#pragma unroll
        for (int it = 0; it < 2; ++it) {
          int f = tid + it * SG_THREADS;  // 512 float4 per tile
          int m = f / 4, kq = (f % 4) * 4;
          float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
          int gm = m0 + m, gk = k0 + kq;
          if (gm < M && gk < k_end) {
            if (gk + 3 < k_end) v = *reinterpret_cast<const float4*>(A + (long long)gm * lda + gk);
            else {
              const float* p = A + (long long)gm * lda + gk;
              v.x = p[0]; if (gk + 1 < k_end) v.y = p[1]; if (gk + 2 < k_end) v.z = p[2];
            }
          }
          As[kq + 0][m] = v.x; As[kq + 1][m] = v.y; As[kq + 2][m] = v.z; As[kq + 3][m] = v.w;
        }
      } else {
#pragma unroll
        for (int it = 0; it < 8; ++it) {
          int e = tid + it * SG_THREADS;
          int m = e / SG_BK, kk = e % SG_BK;
          int gm = m0 + m, gk = k0 + kk;
          As[kk][m] = (gm < M && gk < k_end) ? A[(long long)gm * lda + gk] : 0.f;
        }
      }
    } else {
#pragma unroll
      for (int it = 0; it < 8; ++it) {
        int e = tid + it * SG_THREADS;
        int kk = e / SG_BM, m = e % SG_BM;
        int gm = m0 + m, gk = k0 + kk;
        As[kk][m] = (gm < M && gk < k_end) ? A[(long long)gk * lda + gm] : 0.f;
      }
    }
    // ---- load B tile -> Bs[k][n]
    if (TB) {
      if (vecB) {
#pragma unroll
        for (int it = 0; it < BN / 64; ++it) {
          int f = tid + it * SG_THREADS;
          int n = f / 4, kq = (f % 4) * 4;
          float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
          int gn = n0 + n, gk = k0 + kq;
          if (gn < N && gk < k_end) {
            if (gk + 3 < k_end) v = *reinterpret_cast<const float4*>(B + (long long)gn * ldb + gk);
            else {
              const float* p = B + (long long)gn * ldb + gk;
              v.x = p[0]; if (gk + 1 < k_end) v.y = p[1]; if (gk + 2 < k_end) v.z = p[2];
            }
          }
          Bs[kq + 0][n] = v.x; Bs[kq + 1][n] = v.y; Bs[kq + 2][n] = v.z; Bs[kq + 3][n] = v.w;
        }
      } else {
#pragma unroll
        for (int it = 0; it < BN / 16; ++it) {
          int e = tid + it * SG_THREADS;
          int n = e / SG_BK, kk = e % SG_BK;
          int gn = n0 + n, gk = k0 + kk;
          Bs[kk][n] = (gn < N && gk < k_end) ? B[(long long)gn * ldb + gk] : 0.f;
        }
      }
    } else {
#pragma unroll
      for (int it = 0; it < BN / 16; ++it) {
        int e = tid + it * SG_THREADS;
        int kk = e / BN, n = e % BN;
        int gn = n0 + n, gk = k0 + kk;
        Bs[kk][n] = (gn < N && gk < k_end) ? B[(long long)gk * ldb + gn] : 0.f;
      }
    }
    __syncthreads();

    if (kmax == SG_BK) {
#pragma unroll
      for (int kk = 0; kk < SG_BK; ++kk) {
        float a[8], b[TN];
        *reinterpret_cast<float4*>(a) = *reinterpret_cast<const float4*>(&As[kk][ty * 8]);
        *reinterpret_cast<float4*>(a + 4) = *reinterpret_cast<const float4*>(&As[kk][ty * 8 + 4]);
        *reinterpret_cast<float4*>(b) = *reinterpret_cast<const float4*>(&Bs[kk][tx * TN]);
        if (TN == 8) *reinterpret_cast<float4*>(b + 4) = *reinterpret_cast<const float4*>(&Bs[kk][tx * TN + 4]);
#pragma unroll
        for (int i = 0; i < 8; ++i)
#pragma unroll
          for (int j = 0; j < TN; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
      }
    } else {
      for (int kk = 0; kk < kmax; ++kk) {
        float a[8], b[TN];
#pragma unroll
        for (int i = 0; i < 8; ++i) a[i] = As[kk][ty * 8 + i];
#pragma unroll
        for (int j = 0; j < TN; ++j) b[j] = Bs[kk][tx * TN + j];
#pragma unroll
        for (int i = 0; i < 8; ++i)
#pragma unroll
          for (int j = 0; j < TN; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
      }
    }
    __syncthreads();
  }

#pragma unroll
  for (int i = 0; i < 8; ++i) {
    int gm = m0 + ty * 8 + i;
    if (gm >= M) continue;
#pragma unroll
    for (int j = 0; j < TN; ++j) {
      int gn = n0 + tx * TN + j;
      if (gn < N) epi(gm, gn, acc[i][j], (int)blockIdx.z);
    }
  }
}

struct EpiStore {  // C[m*ldc + n] = v
  float* C; long long ldc;
  __device__ __forceinline__ void operator()(int m, int n, float v, int) const { C[(long long)m * ldc + n] = v; }
};

struct EpiStoreSplit {  // partial[z][m*ldc + n] = v   (deterministic split-K; reduced by a second kernel)
  float* C; long long ldc; long long split_stride;
  __device__ __forceinline__ void operator()(int m, int n, float v, int z) const {
    C[(long long)z * split_stride + (long long)m * ldc + n] = v;
  }
};

static inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

// How launch_sgemm cuts K for a request of `splits` ranges: kps indices per range (a multiple of SG_BK) and the number of
// ranges it runs, which is never more than requested.
struct SgemmSplit { int kps, splits; };
static inline SgemmSplit sgemm_split(int K, int splits) {
  if (splits <= 1 || K <= 0) return {K > 0 ? K : SG_BK, 1};
  const int kps = (int)(ceil_div(ceil_div(K, splits), SG_BK) * SG_BK);
  return {kps, (int)ceil_div(K, kps)};
}

// Split count for a reduction over the batch (K = B): ranges of about 4096 rows, at most 16.
static inline int sgemm_batch_splits(long long B) { long long z = ceil_div(B, 4096); return (int)(z < 1 ? 1 : (z > 16 ? 16 : z)); }

// Host launcher.  splits > 1 => K is cut as sgemm_split says, blockIdx.z = range.
template <bool TA, bool TB, class Epi>
static inline int launch_sgemm(const float* A, long long lda, const float* B, long long ldb, int M, int N, int K,
                               int splits, Epi epi, cudaStream_t st) {
  if (M <= 0 || N <= 0) return TFRS_OK;
  const SgemmSplit sp = sgemm_split(K, splits);
  const int kps = sp.kps;
  splits = sp.splits;
  bool vecA = !TA && (lda % 4 == 0) && aligned16(A);
  bool vecB = TB && (ldb % 4 == 0) && aligned16(B);
  const bool skinny = N <= 64;  // 64-column tiles: no half-empty tiles for the [*, d] outputs of the backward passes
  dim3 grid((unsigned)ceil_div(N, skinny ? 64 : SG_BN), (unsigned)ceil_div(M, SG_BM), (unsigned)splits);
  if (grid.y > 65535) { set_error("sgemm: M too large (%d)", M); return TFRS_ERR_UNSUPPORTED; }
  if (skinny) sgemm_kernel<TA, TB, 64, Epi><<<grid, SG_THREADS, 0, st>>>(A, lda, B, ldb, M, N, K, kps, vecA, vecB, epi);
  else sgemm_kernel<TA, TB, SG_BN, Epi><<<grid, SG_THREADS, 0, st>>>(A, lda, B, ldb, M, N, K, kps, vecA, vecB, epi);
  TFRS_LAUNCH_CHECK();
  return TFRS_OK;
}

// Exact split-K:  out[M,N] (contiguous) = the per-range chains of launch_sgemm summed in fixed order (range ascending).
// `partial` holds `splits` x M x N floats; the launch may use fewer ranges, never more.
template <bool TA, bool TB>
static inline int launch_sgemm_split_k(const float* A, long long lda, const float* B, long long ldb, int M, int N, int K, int splits,
                                       float* partial, float* out, cudaStream_t st) {
  const long long elems = (long long)M * N;
  const int rc = launch_sgemm<TA, TB>(A, lda, B, ldb, M, N, K, splits, EpiStoreSplit{partial, N, elems}, st);
  if (rc) return rc;
  return reduce_parts(partial, M, N, sgemm_split(K, splits).splits, out, N, st);
}

}  // namespace tfrs
