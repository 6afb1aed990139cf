// batch_norm.cu -- K24: tf.keras.layers.BatchNormalization over the rows of x [N, d] (the statistics are per column).
// Every kernel has the same layout: a CTA of 8 warps owns 32 columns (lane = column) and a fixed chunk of rows (warp w
// takes rows r0 + w, r0 + w + 8, ...), so a warp reads 128 contiguous bytes per row.  The chunk is a function of (N, d)
// alone, and every sum runs in a fixed order (rows within a warp ascending, then the 8 warps, then the chunks), so every
// output is bitwise reproducible on any device.  There are no float atomics.
//   training forward: (1) each CTA sums t = x - K, t^2 and the weights over its chunk's kept rows, K = the chunk's first
//     kept row (a shift, so the fp32 sums stay accurate when |mean| >> std; a dropped row's value never enters them, not
//     even as the shift), and keeps K with its sums; (2) per column, the chunk partials fold in fp64:
//     n = sum n_p, mean = sum (n_p K_p + S1_p) / n, M2 = sum S2_p + 2 (K_p - mean) S1_p + n_p (K_p - mean)^2, var =
//     M2 / n; the mean is kept as the fp32 pair hi = f32(mean), lo = f32(mean - hi); the moving statistics are updated
//     here; (3) y = ((x - hi) - lo) rstd gamma + beta.  Three launches.
//   inference forward: y = (x - mm) rstd_mv gamma + beta.  One launch.
//   backward: (1) per-CTA partials of sum dy xhat and sum dy over all rows (inference also writes dx = dy gamma
//     rstd_mv); (2) the partials fold in fp32, chunk ascending, into (dgamma, dbeta); (3) training only: dx = gamma rstd
//     (dy - w (S1 + xhat S2) / n).  Three launches in training, two at inference.
#include "common.cuh"

namespace tfrs {

constexpr int BN_THREADS = 256;
constexpr int BN_WARPS = BN_THREADS / 32;
constexpr long long BN_MIN_CHUNK = 32;      // rows per CTA, at least
constexpr long long BN_TARGET_CTAS = 2048;  // row chunks x column tiles, about two waves of 8 CTAs per SM on an H100

struct BnRows {
  long long c, r0, r1;
  int warp, lane;
};

__device__ __forceinline__ BnRows bn_rows(long long N, long long chunk) {
  BnRows b;
  b.lane = threadIdx.x % 32;
  b.warp = threadIdx.x / 32;
  b.c = (long long)blockIdx.x * 32 + b.lane;
  b.r0 = (long long)blockIdx.y * chunk;
  b.r1 = b.r0 + chunk < N ? b.r0 + chunk : N;
  return b;
}

// sum over the 8 warps of v, warp ascending; every thread gets the column's total
template <typename T>
__device__ __forceinline__ T bn_warps_sum(T v, T (*sh)[32], int warp, int lane) {
  __syncthreads();
  sh[warp][lane] = v;
  __syncthreads();
  T s = sh[0][lane];
#pragma unroll
  for (int w = 1; w < BN_WARPS; ++w) s += sh[w][lane];
  return s;
}

// (1) part [parts, 3, d] = (sum w (x - K), sum w (x - K)^2, K) and count [parts] = sum w over the chunk, K = x at the
// chunk's first kept row (0 when the chunk keeps no row)
__global__ void __launch_bounds__(BN_THREADS)
bn_stats_kernel(const float* __restrict__ x, const void* __restrict__ mask, int mk, long long N, long long d,
                long long chunk, float* __restrict__ part, float* __restrict__ count) {
  __shared__ float sh[BN_WARPS][32];
  __shared__ int first;
  const BnRows b = bn_rows(N, chunk);
  // the first kept row: 256 rows at a time, the lowest kept one of the first window that has any
  long long rk = b.r0;
  if (mask) {
    if (threadIdx.x == 0) first = BN_THREADS;
    rk = b.r1;
    for (long long base = b.r0; base < b.r1; base += BN_THREADS) {
      const long long r = base + threadIdx.x;
      const int kept = r < b.r1 && mask_kept(mask, mk, r);
      if (__syncthreads_or(kept)) {
        if (kept) atomicMin(&first, (int)threadIdx.x);
        __syncthreads();
        rk = base + first;
        break;
      }
    }
  }
  float s1 = 0.f, s2 = 0.f, cnt = 0.f, K = 0.f;
  if (b.c < d && rk < b.r1) {
    K = x[rk * d + b.c];
#pragma unroll 4
    for (long long r = b.r0 + b.warp; r < b.r1; r += BN_WARPS) {
      if (!mask || mask_kept(mask, mk, r)) {
        const float t = x[r * d + b.c] - K;
        s1 += t;
        s2 = fmaf(t, t, s2);
        cnt += 1.f;
      }
    }
  }
  s1 = bn_warps_sum(s1, sh, b.warp, b.lane);
  s2 = bn_warps_sum(s2, sh, b.warp, b.lane);
  cnt = bn_warps_sum(cnt, sh, b.warp, b.lane);
  if (b.warp == 0 && b.c < d) {
    float* pp = part + 3 * (long long)blockIdx.y * d + b.c;
    pp[0] = s1;
    pp[d] = s2;
    pp[2 * d] = K;
    if (b.c == 0) count[blockIdx.y] = cnt;
  }
}

// (2) stats [3 d + 1] = (hi [d], lo [d], rstd [d], n); the moving statistics updated in place (nullable)
__global__ void __launch_bounds__(BN_THREADS)
bn_fold_fwd_kernel(const float* __restrict__ part, const float* __restrict__ count, long long d, int parts, float eps,
                   float decay, float* moving_mean, float* moving_var, float* __restrict__ stats) {
  __shared__ double sh[BN_WARPS][32];
  const int lane = threadIdx.x % 32, warp = threadIdx.x / 32;
  const long long c = (long long)blockIdx.x * 32 + lane;
  double n = 0.0, t1 = 0.0;
  if (c < d)
    for (int p = warp; p < parts; p += BN_WARPS) {
      const float* pp = part + 3ll * p * d + c;
      const double np = count[p];
      n += np;
      t1 += np * (double)pp[2 * d] + (double)pp[0];
    }
  n = bn_warps_sum(n, sh, warp, lane);
  t1 = bn_warps_sum(t1, sh, warp, lane);
  const double mean = n > 0.0 ? t1 / n : 0.0;
  double m2 = 0.0;
  if (c < d)
    for (int p = warp; p < parts; p += BN_WARPS) {
      const float* pp = part + 3ll * p * d + c;
      const double k = (double)pp[2 * d] - mean;
      m2 += (double)pp[d] + 2.0 * k * (double)pp[0] + (double)count[p] * k * k;
    }
  m2 = bn_warps_sum(m2, sh, warp, lane);
  if (warp != 0 || c >= d) return;
  const float hi = (float)mean, lo = (float)(mean - (double)hi);
  const float var = n > 0.0 && m2 > 0.0 ? (float)(m2 / n) : 0.f;
  stats[c] = hi;
  stats[d + c] = lo;
  stats[2 * d + c] = 1.f / sqrtf(var + eps);
  if (c == 0) stats[3 * d] = (float)n;
  if (moving_mean) {
    const float mm = moving_mean[c], mv = moving_var[c];
    moving_mean[c] = __fsub_rn(mm, __fmul_rn(__fsub_rn(mm, __fadd_rn(hi, lo)), decay));
    moving_var[c] = __fsub_rn(mv, __fmul_rn(__fsub_rn(mv, var), decay));
  }
}

// (3) y = ((x - hi) - lo) rstd gamma + beta, from stats (training) or from the moving statistics (inference, which
// also writes the backward's saved (hi, lo, rstd) when `saved` is given)
__global__ void __launch_bounds__(BN_THREADS)
bn_apply_kernel(const float* __restrict__ x, const float* __restrict__ gamma, const float* __restrict__ beta,
                const float* __restrict__ stats, const float* __restrict__ moving_mean,
                const float* __restrict__ moving_var, float eps, long long N, long long d, long long chunk,
                float* __restrict__ y, float* __restrict__ saved) {
  const BnRows b = bn_rows(N, chunk);
  if (b.c >= d) return;
  float hi, lo, rs;
  if (stats) {
    hi = stats[b.c];
    lo = stats[d + b.c];
    rs = stats[2 * d + b.c];
  } else {
    hi = moving_mean[b.c];
    lo = 0.f;
    rs = 1.f / sqrtf(moving_var[b.c] + eps);
    if (saved && blockIdx.y == 0 && b.warp == 0) {
      saved[b.c] = hi;
      saved[d + b.c] = lo;
      saved[2 * d + b.c] = rs;
      if (b.c == 0) saved[3 * d] = 0.f;
    }
  }
  const float g = gamma ? gamma[b.c] : 1.f, be = beta ? beta[b.c] : 0.f;
#pragma unroll 4
  for (long long r = b.r0 + b.warp; r < b.r1; r += BN_WARPS) {
    float t = ((x[r * d + b.c] - hi) - lo) * rs;
    if (gamma) t *= g;
    if (beta) t += be;
    y[r * d + b.c] = t;
  }
}

// backward (1): part [parts, 2, d] = (sum dy xhat, sum dy) over the chunk's rows; at inference also dx = dy gamma rstd
__global__ void __launch_bounds__(BN_THREADS)
bn_bwd_part_kernel(const float* __restrict__ x, const float* __restrict__ gamma, const float* __restrict__ saved,
                   const float* __restrict__ dy, long long N, long long d, long long chunk, float* __restrict__ part,
                   float* __restrict__ dx) {
  __shared__ float sh[BN_WARPS][32];
  const BnRows b = bn_rows(N, chunk);
  float a = 0.f, s = 0.f;
  if (b.c < d) {
    const float hi = saved[b.c], lo = saved[d + b.c], rs = saved[2 * d + b.c];
    const float k = gamma ? __fmul_rn(gamma[b.c], rs) : rs;
#pragma unroll 4
    for (long long r = b.r0 + b.warp; r < b.r1; r += BN_WARPS) {
      const float g = dy[r * d + b.c];
      a = fmaf(g, ((x[r * d + b.c] - hi) - lo) * rs, a);
      s += g;
      if (dx) dx[r * d + b.c] = g * k;
    }
  }
  a = bn_warps_sum(a, sh, b.warp, b.lane);
  s = bn_warps_sum(s, sh, b.warp, b.lane);
  if (b.warp == 0 && b.c < d) {
    part[(2 * (long long)blockIdx.y) * d + b.c] = a;
    part[(2 * (long long)blockIdx.y + 1) * d + b.c] = s;
  }
}

// backward (2): dparams [2, d] = (dgamma, dbeta) = the partials summed in fp32, warp-strided chunks then warp ascending
__global__ void __launch_bounds__(BN_THREADS)
bn_bwd_fold_kernel(const float* __restrict__ part, long long d, int parts, float* __restrict__ dparams) {
  __shared__ float sh[BN_WARPS][32];
  const int lane = threadIdx.x % 32, warp = threadIdx.x / 32;
  const long long c = (long long)blockIdx.x * 32 + lane;
  float a = 0.f, s = 0.f;
  if (c < d)
    for (int p = warp; p < parts; p += BN_WARPS) {
      a += part[2ll * p * d + c];
      s += part[(2ll * p + 1) * d + c];
    }
  a = bn_warps_sum(a, sh, warp, lane);
  s = bn_warps_sum(s, sh, warp, lane);
  if (warp == 0 && c < d) {
    dparams[c] = a;
    dparams[d + c] = s;
  }
}

// backward (3), training: dx = gamma rstd (dy - w (S1 + xhat S2) / n)
__global__ void __launch_bounds__(BN_THREADS)
bn_bwd_dx_kernel(const float* __restrict__ x, const void* __restrict__ mask, int mk, const float* __restrict__ gamma,
                 const float* __restrict__ saved, const float* __restrict__ dparams, const float* __restrict__ dy,
                 long long N, long long d, long long chunk, float* __restrict__ dx) {
  const BnRows b = bn_rows(N, chunk);
  if (b.c >= d) return;
  const float hi = saved[b.c], lo = saved[d + b.c], rs = saved[2 * d + b.c], n = saved[3 * d];
  const float k = gamma ? __fmul_rn(gamma[b.c], rs) : rs;
  const float s2n = n > 0.f ? dparams[b.c] / n : 0.f, s1n = n > 0.f ? dparams[d + b.c] / n : 0.f;
#pragma unroll 4
  for (long long r = b.r0 + b.warp; r < b.r1; r += BN_WARPS) {
    const float g = dy[r * d + b.c];
    const float u = !mask || mask_kept(mask, mk, r) ? g - (s1n + ((x[r * d + b.c] - hi) - lo) * rs * s2n) : g;
    dx[r * d + b.c] = k * u;
  }
}

// row chunk and chunk count: a function of (N, d) alone, so the fold order never depends on the device
static void bn_chunks(long long N, long long d, long long* chunk, long long* parts) {
  long long p = BN_TARGET_CTAS / ceil_div(d, 32);
  if (p < 1) p = 1;
  const long long pmax = ceil_div(N, BN_MIN_CHUNK);
  if (p > pmax) p = pmax;
  *chunk = ceil_div(N, p);
  *parts = ceil_div(N, *chunk);
}

static bool bn_shape_ok(long long N, long long d) { return N >= 1 && d >= 1 && d < (1ll << 31) && N < (1ll << 62) / d; }

}  // namespace tfrs
using namespace tfrs;

extern "C" size_t tfrs_batch_norm_fwd_workspace_bytes(int64_t N, int64_t d) {
  if (!bn_shape_ok(N, d)) return 256;
  long long chunk, parts;
  bn_chunks(N, d, &chunk, &parts);
  return align_up((size_t)parts * 3 * d * 4, 256) + align_up((size_t)parts * 4, 256) + align_up(((size_t)3 * d + 1) * 4, 256);
}

extern "C" int tfrs_batch_norm_fwd_f32(const float* x, const void* mask, int mask_kind, const float* gamma,
                                       const float* beta, int64_t N, int64_t d, int training, double momentum, float eps,
                                       float* moving_mean, float* moving_var, float* y, float* saved, void* ws,
                                       size_t ws_bytes, void* stream) {
  TFRS_CHECK_ARG(bn_shape_ok(N, d), "batch_norm_fwd: bad shape N=%lld d=%lld", (long long)N, (long long)d);
  TFRS_CHECK_ARG(x && y && moving_mean && moving_var, "batch_norm_fwd: NULL pointer");
  TFRS_CHECK_MASK("batch_norm_fwd", mask, mask_kind);
  TFRS_CHECK_ARG(eps >= 0.f, "batch_norm_fwd: epsilon must be >= 0");
  cudaStream_t st = (cudaStream_t)stream;
  long long chunk, parts;
  bn_chunks(N, d, &chunk, &parts);
  const dim3 grid((unsigned)ceil_div(d, 32), (unsigned)parts);
  if (!training) {
    bn_apply_kernel<<<grid, BN_THREADS, 0, st>>>(x, gamma, beta, nullptr, moving_mean, moving_var, eps, N, d, chunk, y,
                                                saved);
    TFRS_LAUNCH_CHECK();
    return TFRS_OK;
  }
  TFRS_CHECK_ARG(momentum >= 0.0 && momentum <= 1.0, "batch_norm_fwd: momentum must be in [0, 1], got %g", momentum);
  if (!ws || ws_bytes < tfrs_batch_norm_fwd_workspace_bytes(N, d)) {
    set_error("batch_norm_fwd: workspace too small");
    return TFRS_ERR_WORKSPACE_TOO_SMALL;
  }
  TFRS_CHECK_ARG((reinterpret_cast<uintptr_t>(ws) & 15) == 0, "batch_norm_fwd: workspace must be 16-byte aligned");
  char* w = static_cast<char*>(ws);
  float* part = reinterpret_cast<float*>(w);
  w += align_up((size_t)parts * 3 * d * 4, 256);
  float* count = reinterpret_cast<float*>(w);
  w += align_up((size_t)parts * 4, 256);
  float* stats = saved ? saved : reinterpret_cast<float*>(w);
  bn_stats_kernel<<<grid, BN_THREADS, 0, st>>>(x, mask, mask_kind, N, d, chunk, part, count);
  TFRS_LAUNCH_CHECK();
  bn_fold_fwd_kernel<<<(unsigned)ceil_div(d, 32), BN_THREADS, 0, st>>>(part, count, d, (int)parts, eps,
                                                                       (float)(1.0 - momentum), moving_mean, moving_var,
                                                                       stats);
  TFRS_LAUNCH_CHECK();
  bn_apply_kernel<<<grid, BN_THREADS, 0, st>>>(x, gamma, beta, stats, nullptr, nullptr, eps, N, d, chunk, y, nullptr);
  TFRS_LAUNCH_CHECK();
  return TFRS_OK;
}

extern "C" size_t tfrs_batch_norm_bwd_workspace_bytes(int64_t N, int64_t d) {
  if (!bn_shape_ok(N, d)) return 256;
  long long chunk, parts;
  bn_chunks(N, d, &chunk, &parts);
  return align_up((size_t)parts * 2 * d * 4, 256);
}

extern "C" int tfrs_batch_norm_bwd_f32(const float* x, const void* mask, int mask_kind, const float* gamma,
                                       const float* saved, const float* dy, int64_t N, int64_t d, int training,
                                       float* dx, float* dparams, void* ws, size_t ws_bytes, void* stream) {
  TFRS_CHECK_ARG(bn_shape_ok(N, d), "batch_norm_bwd: bad shape N=%lld d=%lld", (long long)N, (long long)d);
  TFRS_CHECK_ARG(x && saved && dy && dparams, "batch_norm_bwd: NULL pointer");
  TFRS_CHECK_MASK("batch_norm_bwd", mask, mask_kind);
  if (!ws || ws_bytes < tfrs_batch_norm_bwd_workspace_bytes(N, d)) {
    set_error("batch_norm_bwd: workspace too small");
    return TFRS_ERR_WORKSPACE_TOO_SMALL;
  }
  TFRS_CHECK_ARG((reinterpret_cast<uintptr_t>(ws) & 15) == 0, "batch_norm_bwd: workspace must be 16-byte aligned");
  cudaStream_t st = (cudaStream_t)stream;
  long long chunk, parts;
  bn_chunks(N, d, &chunk, &parts);
  const dim3 grid((unsigned)ceil_div(d, 32), (unsigned)parts);
  float* part = static_cast<float*>(ws);
  bn_bwd_part_kernel<<<grid, BN_THREADS, 0, st>>>(x, gamma, saved, dy, N, d, chunk, part, training ? nullptr : dx);
  TFRS_LAUNCH_CHECK();
  bn_bwd_fold_kernel<<<(unsigned)ceil_div(d, 32), BN_THREADS, 0, st>>>(part, d, (int)parts, dparams);
  TFRS_LAUNCH_CHECK();
  if (!training || !dx) return TFRS_OK;
  bn_bwd_dx_kernel<<<grid, BN_THREADS, 0, st>>>(x, mask, mask_kind, gamma, saved, dparams, dy, N, d, chunk, dx);
  TFRS_LAUNCH_CHECK();
  return TFRS_OK;
}
