// features.cu -- K17: the numeric feature columns and the pooling of the reference's context-feature towers:
// layers.Discretization (TF's Bucketize), layers.Normalization (call and adapt) and layers.GlobalAveragePooling1D with a
// mask.  Every result is deterministic: no float atomics, fixed summation orders, one IEEE operation per step.
//
//   tfrs_bucketize            one element per thread (grid-stride), a binary search over the float32 boundaries, which
//                             are staged in shared memory when they fit in 48 KB.
//   tfrs_normalize            elementwise, with the int / float64 -> float32 conversion fused in.
//   tfrs_normalization_adapt  one thread per (batch, channel) for every batch's moments, then one thread per channel
//                             folds the batches in order into the device state; a single batch takes one fused launch.
//   tfrs_mean_pool_fwd / bwd  one thread per (row, column): a sequential sum over t.
#include "common.cuh"

namespace tfrs {

constexpr int FT_THREADS = 256;
constexpr int64_t FT_SMEM_BOUNDS = 12288;   // 48 KB of float32 boundaries: the default dynamic shared memory limit
constexpr float FT_EPSILON = 1e-7f;         // keras.backend.epsilon()

template <typename T> __device__ __forceinline__ float ft_f32(T x);
template <> __device__ __forceinline__ float ft_f32<int32_t>(int32_t x) { return __int2float_rn(x); }
template <> __device__ __forceinline__ float ft_f32<long long>(long long x) { return __ll2float_rn(x); }
template <> __device__ __forceinline__ float ft_f32<float>(float x) { return x; }
template <> __device__ __forceinline__ float ft_f32<double>(double x) { return __double2float_rn(x); }

// x < b as Bucketize compares: integers and float32 as float32, float64 as double
template <typename T> __device__ __forceinline__ bool ft_less(T x, float b) { return ft_f32(x) < b; }
template <> __device__ __forceinline__ bool ft_less<double>(double x, float b) { return x < (double)b; }

// ---- bucketize ------------------------------------------------------------------------------------------------------
template <typename T, bool SMEM>
__global__ void __launch_bounds__(FT_THREADS)
ft_bucketize_kernel(const T* __restrict__ x, long long n, const float* __restrict__ bounds, int nb,
                    long long* __restrict__ out) {
  extern __shared__ float sb[];
  const float* b = bounds;
  if (SMEM) {
    for (int k = threadIdx.x; k < nb; k += FT_THREADS) sb[k] = bounds[k];
    __syncthreads();
    b = sb;
  }
  for (long long i = (long long)blockIdx.x * FT_THREADS + threadIdx.x; i < n; i += (long long)gridDim.x * FT_THREADS) {
    const T v = x[i];
    int lo = 0, hi = nb;                  // std::upper_bound: the first boundary above v
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (ft_less(v, SMEM ? b[mid] : __ldg(b + mid))) hi = mid;
      else lo = mid + 1;
    }
    out[i] = lo;
  }
}

// ---- normalize ------------------------------------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(FT_THREADS)
ft_normalize_kernel(const T* __restrict__ x, long long n, long long C, const float* __restrict__ mean,
                    const float* __restrict__ var, int invert, float* __restrict__ out) {
  for (long long i = (long long)blockIdx.x * FT_THREADS + threadIdx.x; i < n; i += (long long)gridDim.x * FT_THREADS) {
    const long long c = C == 1 ? 0 : i % C;
    const float v = ft_f32(x[i]), m = __ldg(mean + c);
    const float s = __fsqrt_rn(__ldg(var + c));
    const float sd = s < FT_EPSILON ? FT_EPSILON : s;     // tf.maximum: a NaN stays NaN
    out[i] = invert ? __fadd_rn(m, __fmul_rn(v, sd)) : __fdiv_rn(__fsub_rn(v, m), sd);
  }
}

// ---- adapt ----------------------------------------------------------------------------------------------------------
// The moments of channel c over rows [r0, r1) of x [N, R]: float32 of the float64 row-major sums, over the count.
template <typename T>
__device__ __forceinline__ void ft_moments(const T* __restrict__ x, long long R, long long C, long long r0, long long r1,
                                           long long c, float* m, float* v) {
  const double cnt = (double)((r1 - r0) * (R / C));
  double s = 0.0;
  for (long long r = r0; r < r1; ++r)
    for (long long e = c; e < R; e += C) s += (double)ft_f32(x[r * R + e]);
  const float mf = (float)(s / cnt);
  double q = 0.0;
  for (long long r = r0; r < r1; ++r)
    for (long long e = c; e < R; e += C) {
      const float d = __fsub_rn(ft_f32(x[r * R + e]), mf);
      q += (double)__fmul_rn(d, d);
    }
  *m = mf;
  *v = (float)(q / cnt);
}

// Keras's Normalization.update_state merge of one batch (mean mb, variance vb, count nb) into (mean, var, total).
__device__ __forceinline__ void ft_merge(float& mean, float& var, long long& total, float mb, float vb, long long nb) {
  total += nb;
  const float w = __fdiv_rn(__ll2float_rn(nb), __ll2float_rn(total));
  const float ew = __fsub_rn(1.f, w);
  const float nm = __fadd_rn(__fmul_rn(mean, ew), __fmul_rn(mb, w));
  const float d0 = __fsub_rn(mean, nm), d1 = __fsub_rn(mb, nm);
  const float a = __fmul_rn(__fadd_rn(var, __fmul_rn(d0, d0)), ew);
  const float b = __fmul_rn(__fadd_rn(vb, __fmul_rn(d1, d1)), w);
  var = __fadd_rn(a, b);
  mean = nm;
}

template <typename T>
__global__ void __launch_bounds__(FT_THREADS)
ft_batch_moments_kernel(const T* __restrict__ x, long long N, long long R, long long C, long long batch_rows,
                        long long nbatch, float* __restrict__ stats) {
  const long long i = (long long)blockIdx.x * FT_THREADS + threadIdx.x;
  if (i >= nbatch * C) return;
  const long long k = i / C, c = i % C;
  const long long r0 = k * batch_rows, r1 = min(N, r0 + batch_rows);
  ft_moments(x, R, C, r0, r1, c, stats + 2 * k * C + c, stats + (2 * k + 1) * C + c);
}

// One block: thread c folds channels c, c + FT_THREADS, ...; the count is written once every thread has read it.
__global__ void __launch_bounds__(FT_THREADS)
ft_fold_kernel(const float* __restrict__ stats, long long N, long long R, long long C, long long batch_rows,
               long long nbatch, float* __restrict__ state, long long* __restrict__ count) {
  const long long total0 = *count;
  long long total = total0;
  for (long long c = threadIdx.x; c < C; c += FT_THREADS) {
    float mean = state[c], var = state[C + c];
    total = total0;
    for (long long k = 0; k < nbatch; ++k) {
      const long long rows = min(N, (k + 1) * batch_rows) - k * batch_rows;
      ft_merge(mean, var, total, stats[2 * k * C + c], stats[(2 * k + 1) * C + c], rows * (R / C));
    }
    state[c] = mean;
    state[C + c] = var;
  }
  __syncthreads();
  if (threadIdx.x == 0) *count = total;
}

// One block, one batch: the moments and the merge of each channel in one thread.
template <typename T>
__global__ void __launch_bounds__(FT_THREADS)
ft_update_kernel(const T* __restrict__ x, long long N, long long R, long long C, float* __restrict__ state,
                 long long* __restrict__ count) {
  const long long total0 = *count;
  long long total = total0;
  for (long long c = threadIdx.x; c < C; c += FT_THREADS) {
    float mb, vb, mean = state[c], var = state[C + c];
    ft_moments(x, R, C, 0, N, c, &mb, &vb);
    total = total0;
    ft_merge(mean, var, total, mb, vb, N * (R / C));
    state[c] = mean;
    state[C + c] = var;
  }
  __syncthreads();
  if (threadIdx.x == 0) *count = total;
}

// ---- masked mean pooling --------------------------------------------------------------------------------------------
template <typename M>
__global__ void __launch_bounds__(FT_THREADS)
ft_pool_fwd_kernel(const float* __restrict__ x, long long B, long long T, long long d, long long sb, long long st,
                   long long sd, const M* __restrict__ mask, float* __restrict__ out) {
  const long long i = (long long)blockIdx.x * FT_THREADS + threadIdx.x;
  if (i >= B * d) return;
  const long long b = i / d, k = i % d;
  const float* xp = x + b * sb + k * sd;
  float s = 0.f, c = 0.f;
  for (long long t = 0; t < T; ++t) {
    if (mask) {
      const float m = mask_kept<M>(mask, b * T + t) ? 1.f : 0.f;
      s = __fadd_rn(s, __fmul_rn(__ldg(xp + t * st), m));
      c = __fadd_rn(c, m);
    } else {
      s = __fadd_rn(s, __ldg(xp + t * st));
    }
  }
  out[i] = __fdiv_rn(s, mask ? c : (float)T);
}

template <typename M>
__global__ void __launch_bounds__(FT_THREADS)
ft_pool_bwd_kernel(const float* __restrict__ g, long long B, long long T, long long d, const M* __restrict__ mask,
                   float* __restrict__ dx) {
  const long long i = (long long)blockIdx.x * FT_THREADS + threadIdx.x;
  if (i >= B * d) return;
  const long long b = i / d, k = i % d;
  float c = (float)T;
  if (mask) {
    c = 0.f;
    for (long long t = 0; t < T; ++t) c = __fadd_rn(c, mask_kept<M>(mask, b * T + t) ? 1.f : 0.f);
  }
  const float q = __fdiv_rn(g[i], c);
  float* dp = dx + b * T * d + k;
  for (long long t = 0; t < T; ++t) dp[t * d] = mask ? __fmul_rn(q, mask_kept<M>(mask, b * T + t) ? 1.f : 0.f) : q;
}

template <typename M>
static int ft_pool(const float* x, long long B, long long T, long long d, long long sb, long long st, long long sd,
                   const void* mask, float* out, bool bwd, cudaStream_t s) {
  const unsigned grid = (unsigned)ceil_div(B * d, FT_THREADS);
  if (bwd) ft_pool_bwd_kernel<M><<<grid, FT_THREADS, 0, s>>>(x, B, T, d, (const M*)mask, out);
  else ft_pool_fwd_kernel<M><<<grid, FT_THREADS, 0, s>>>(x, B, T, d, sb, st, sd, (const M*)mask, out);
  TFRS_LAUNCH_CHECK();
  return TFRS_OK;
}

static int ft_pool_any(const float* x, long long B, long long T, long long d, long long sb, long long st, long long sd,
                       const void* mask, int mask_kind, float* out, bool bwd, cudaStream_t s) {
  const char* what = bwd ? "mean_pool_bwd" : "mean_pool_fwd";
  TFRS_CHECK_ARG(B >= 0 && T >= 0 && d >= 0 && B * d < (1ll << 40) && B * T < (1ll << 40) && B * T * d < (1ll << 46),
                 "%s: bad shape [%lld, %lld, %lld]", what, B, T, d);
  TFRS_CHECK_MASK(what, mask, mask_kind);
  if (B * d == 0) return TFRS_OK;
  // an empty time axis leaves x (forward) or dx (backward) empty, and possibly NULL
  TFRS_CHECK_ARG(bwd ? x && (out || T == 0) : out && (x || T == 0), "%s: NULL input or output", what);
  return mask_dispatch(mask, mask_kind,
                       [&](auto m) { return ft_pool<decltype(m)>(x, B, T, d, sb, st, sd, mask, out, bwd, s); });
}

static bool ft_kind(int kind) { return kind == TFRS_I32 || kind == TFRS_I64 || kind == TFRS_F32 || kind == TFRS_F64; }

// Calls f(T{}) with T the C++ type of a value kind.
template <typename F>
static int ft_dispatch(int kind, F f) {
  switch (kind) {
    case TFRS_I32: return f(int32_t{});
    case TFRS_I64: return f((long long)0);
    case TFRS_F32: return f(0.f);
    default: return f(0.0);
  }
}

static size_t ft_adapt_ws(long long N, long long C, long long batch_rows) {
  return N <= batch_rows ? 0 : align_up((size_t)ceil_div(N, batch_rows) * 2 * (size_t)C * 4, 256);
}

}  // namespace tfrs

using namespace tfrs;

extern "C" int tfrs_bucketize(const void* x, int kind, int64_t n, const float* bounds, int64_t nb, int64_t* out,
                              void* stream) {
  TFRS_CHECK_ARG(ft_kind(kind), "bucketize: values must be I32, I64, F32 or F64");
  TFRS_CHECK_ARG(n >= 0 && nb >= 0 && nb < (1ll << 31), "bucketize: bad n = %lld or nb = %lld", (long long)n,
                 (long long)nb);
  if (n == 0) return TFRS_OK;
  TFRS_CHECK_ARG(x && out && (nb == 0 || bounds), "bucketize: NULL values, boundaries or out");
  cudaStream_t st = (cudaStream_t)stream;
  const unsigned grid = elementwise_grid(n);
  long long* o = reinterpret_cast<long long*>(out);
  return ft_dispatch(kind, [&](auto t) -> int {
    using T = decltype(t);
    if (nb <= FT_SMEM_BOUNDS)
      ft_bucketize_kernel<T, true><<<grid, FT_THREADS, nb * 4, st>>>((const T*)x, n, bounds, (int)nb, o);
    else
      ft_bucketize_kernel<T, false><<<grid, FT_THREADS, 0, st>>>((const T*)x, n, bounds, (int)nb, o);
    TFRS_LAUNCH_CHECK();
    return TFRS_OK;
  });
}

extern "C" int tfrs_normalize(const void* x, int kind, int64_t n, int64_t C, const float* mean, const float* var,
                              int invert, float* out, void* stream) {
  TFRS_CHECK_ARG(ft_kind(kind), "normalize: values must be I32, I64, F32 or F64");
  TFRS_CHECK_ARG(n >= 0 && C >= 1 && n % C == 0, "normalize: bad n = %lld or C = %lld", (long long)n, (long long)C);
  if (n == 0) return TFRS_OK;
  TFRS_CHECK_ARG(x && mean && var && out, "normalize: NULL values, statistics or out");
  cudaStream_t st = (cudaStream_t)stream;
  const unsigned grid = elementwise_grid(n);
  return ft_dispatch(kind, [&](auto t) -> int {
    using T = decltype(t);
    ft_normalize_kernel<T><<<grid, FT_THREADS, 0, st>>>((const T*)x, n, C, mean, var, invert ? 1 : 0, out);
    TFRS_LAUNCH_CHECK();
    return TFRS_OK;
  });
}

extern "C" size_t tfrs_normalization_adapt_workspace_bytes(int64_t N, int64_t C, int64_t batch_rows) {
  if (N < 0 || C < 1 || batch_rows < 1) return 0;
  return ft_adapt_ws(N, C, batch_rows);
}

extern "C" int tfrs_normalization_adapt(const void* x, int kind, int64_t N, int64_t R, int64_t C, int64_t batch_rows,
                                        float* state, int64_t* count, void* ws, size_t ws_bytes, void* stream) {
  TFRS_CHECK_ARG(ft_kind(kind), "normalization_adapt: values must be I32, I64, F32 or F64");
  TFRS_CHECK_ARG(N >= 0 && R >= 1 && C >= 1 && R % C == 0 && batch_rows >= 1 && N * R < (1ll << 46) &&
                     C <= (1ll << 30), "normalization_adapt: bad N = %lld, R = %lld, C = %lld or batch_rows = %lld",
                 (long long)N, (long long)R, (long long)C, (long long)batch_rows);
  if (N == 0) return TFRS_OK;
  TFRS_CHECK_ARG(x && state && count, "normalization_adapt: NULL values, state or count");
  TFRS_CHECK_ARG(ws_bytes >= ft_adapt_ws(N, C, batch_rows) && (ws || N <= batch_rows),
                 "normalization_adapt: workspace too small");
  cudaStream_t st = (cudaStream_t)stream;
  long long* cnt = reinterpret_cast<long long*>(count);
  return ft_dispatch(kind, [&](auto t) -> int {
    using T = decltype(t);
    if (N <= batch_rows) {
      ft_update_kernel<T><<<1, FT_THREADS, 0, st>>>((const T*)x, N, R, C, state, cnt);
      TFRS_LAUNCH_CHECK();
      return TFRS_OK;
    }
    const long long nbatch = ceil_div(N, batch_rows);
    float* stats = reinterpret_cast<float*>(ws);
    ft_batch_moments_kernel<T><<<(unsigned)ceil_div(nbatch * C, FT_THREADS), FT_THREADS, 0, st>>>(
        (const T*)x, N, R, C, batch_rows, nbatch, stats);
    TFRS_LAUNCH_CHECK();
    ft_fold_kernel<<<1, FT_THREADS, 0, st>>>(stats, N, R, C, batch_rows, nbatch, state, cnt);
    TFRS_LAUNCH_CHECK();
    return TFRS_OK;
  });
}

extern "C" int tfrs_mean_pool_fwd(const float* x, int64_t B, int64_t T, int64_t d, int64_t sb, int64_t st, int64_t sd,
                                  const void* mask, int mask_kind, float* out, void* stream) {
  return ft_pool_any(x, B, T, d, sb, st, sd, mask, mask_kind, out, false, (cudaStream_t)stream);
}

extern "C" int tfrs_mean_pool_bwd(const float* g, int64_t B, int64_t T, int64_t d, const void* mask, int mask_kind,
                                  float* dx, void* stream) {
  return ft_pool_any(g, B, T, d, 0, 0, 0, mask, mask_kind, dx, true, (cudaStream_t)stream);
}
