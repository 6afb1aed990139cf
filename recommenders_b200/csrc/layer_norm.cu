// layer_norm.cu -- K22: tf.keras.layers.LayerNormalization over the last axis.  One warp per row: each lane takes the
// columns lane, lane + 32, ... and the row sums are fp32 lane sums followed by a butterfly, so every lane holds them.
//   forward: pass 1 gives hi = sum(x) / d; pass 2 sums x - hi and (x - hi)^2, so lo = sum(x - hi) / d and var =
//     sum((x - hi)^2) / d - lo^2 (the corrected two-pass variance, never E[x^2] - E[x]^2); then y from
//     xhat = ((x - hi) - lo) rstd.  The mean is kept as the pair hi + lo: x - hi is exact for x near hi, so a row with
//     mean 1e4 and std 1 loses nothing to the 1e-3 spacing of fp32 at 1e4.  (hi, lo) and rstd are saved for the
//     backward.  One launch.
//   backward: each CTA owns a fixed chunk of rows.  Its warps write dx row by row; then each thread owns columns and
//     sums dy * xhat and dy over the chunk's rows in order into the CTA's partial [2, d]; reduce_parts (reduce.cu) folds
//     the partials, CTA ascending.  Two launches, no atomics, bitwise reproducible.
#include "common.cuh"

namespace tfrs {

constexpr int LN_THREADS = 256;
constexpr int LN_WARPS = LN_THREADS / 32;
constexpr long long LN_MIN_CHUNK = 16;      // rows per backward CTA, at least
constexpr long long LN_MAX_PARTS = 1024;    // backward CTAs (partials) at most

__device__ __forceinline__ float warp_sum(float x) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) x += __shfl_xor_sync(0xffffffffu, x, o);
  return x;
}

__global__ void __launch_bounds__(LN_THREADS)
ln_fwd_kernel(const float* __restrict__ x, const float* __restrict__ gamma, const float* __restrict__ beta, long long N,
              long long d, float eps, float* __restrict__ y, float* __restrict__ mean, float* __restrict__ rstd) {
  const int lane = threadIdx.x % 32;
  const long long stride = (long long)gridDim.x * LN_WARPS;
  for (long long r = (long long)blockIdx.x * LN_WARPS + threadIdx.x / 32; r < N; r += stride) {
    const float* xr = x + r * d;
    float s = 0.f;
    for (long long c = lane; c < d; c += 32) s += xr[c];
    const float hi = warp_sum(s) / (float)d;
    float s1 = 0.f, s2 = 0.f;
    for (long long c = lane; c < d; c += 32) {
      const float t = xr[c] - hi;
      s1 += t;
      s2 = fmaf(t, t, s2);
    }
    const float lo = warp_sum(s1) / (float)d;
    const float var = fmaxf(warp_sum(s2) / (float)d - lo * lo, 0.f);
    const float rs = 1.f / sqrtf(var + eps);
    float* yr = y + r * d;
    for (long long c = lane; c < d; c += 32) {
      float t = ((xr[c] - hi) - lo) * rs;
      if (gamma) t *= gamma[c];
      if (beta) t += beta[c];
      yr[c] = t;
    }
    if (mean && lane == 0) {
      mean[2 * r] = hi;
      mean[2 * r + 1] = lo;
      rstd[r] = rs;
    }
  }
}

__global__ void __launch_bounds__(LN_THREADS)
ln_bwd_kernel(const float* __restrict__ x, const float* __restrict__ gamma, const float* __restrict__ mean,
              const float* __restrict__ rstd, const float* __restrict__ dy, long long N, long long d, long long chunk,
              float* __restrict__ dx, float* __restrict__ part) {
  const int lane = threadIdx.x % 32;
  const long long r0 = (long long)blockIdx.x * chunk, r1 = r0 + chunk < N ? r0 + chunk : N;
  const float inv_d = 1.f / (float)d;
  if (dx)
    for (long long r = r0 + threadIdx.x / 32; r < r1; r += LN_WARPS) {
      const float* xr = x + r * d;
      const float* gr = dy + r * d;
      const float hi = mean[2 * r], lo = mean[2 * r + 1], rs = rstd[r];
      float sg = 0.f, sgx = 0.f;
      for (long long c = lane; c < d; c += 32) {
        const float g = gamma ? __fmul_rn(gr[c], gamma[c]) : gr[c];   // rounded, never contracted into g - mg
        sg += g;
        sgx = fmaf(g, ((xr[c] - hi) - lo) * rs, sgx);
      }
      const float mg = warp_sum(sg) * inv_d, mgx = warp_sum(sgx) * inv_d;
      float* dr = dx + r * d;
      for (long long c = lane; c < d; c += 32) {
        const float g = gamma ? __fmul_rn(gr[c], gamma[c]) : gr[c];   // rounded, never contracted into g - mg
        dr[c] = rs * (g - mg - ((xr[c] - hi) - lo) * rs * mgx);
      }
    }
  if (!part) return;
  float* pr = part + (long long)blockIdx.x * 2 * d;
  for (long long c = threadIdx.x; c < d; c += LN_THREADS) {
    float a = 0.f, b = 0.f;
    for (long long r = r0; r < r1; ++r) {
      const float g = dy[r * d + c];
      a = fmaf(g, ((x[r * d + c] - mean[2 * r]) - mean[2 * r + 1]) * rstd[r], a);
      b += g;
    }
    pr[c] = a;
    pr[d + c] = b;
  }
}

// rows per backward CTA and the CTA count: a function of N alone, so the fold order never depends on the device
static void ln_chunks(long long N, long long* chunk, long long* parts) {
  long long c = ceil_div(N, LN_MAX_PARTS);
  *chunk = c < LN_MIN_CHUNK ? LN_MIN_CHUNK : c;
  *parts = ceil_div(N, *chunk);
}

}  // namespace tfrs
using namespace tfrs;

extern "C" int tfrs_layer_norm_fwd_f32(const float* x, const float* gamma, const float* beta, int64_t N, int64_t d,
                                       float eps, float* y, float* mean, float* rstd, void* stream) {
  TFRS_CHECK_ARG(N >= 0 && d >= 1 && d < (1ll << 31), "layer_norm_fwd: bad shape N=%lld d=%lld", (long long)N,
                 (long long)d);
  TFRS_CHECK_ARG(!mean == !rstd, "layer_norm_fwd: mean and rstd are saved together");
  TFRS_CHECK_ARG(eps >= 0.f, "layer_norm_fwd: epsilon must be >= 0");
  if (N == 0) return TFRS_OK;
  TFRS_CHECK_ARG(x && y, "layer_norm_fwd: NULL pointer");
  const long long want = ceil_div(N, LN_WARPS), cap = (long long)sm_count() * 16;
  ln_fwd_kernel<<<(unsigned)(want < cap ? want : cap), LN_THREADS, 0, (cudaStream_t)stream>>>(x, gamma, beta, N, d, eps,
                                                                                            y, mean, rstd);
  TFRS_LAUNCH_CHECK();
  return TFRS_OK;
}

extern "C" size_t tfrs_layer_norm_bwd_workspace_bytes(int64_t N, int64_t d) {
  if (N <= 0 || d <= 0) return 256;
  long long chunk, parts;
  ln_chunks(N, &chunk, &parts);
  const size_t bytes = align_up((size_t)parts * 2 * d * 4, 256);
  return bytes < 256 ? 256 : bytes;
}

extern "C" int tfrs_layer_norm_bwd_f32(const float* x, const float* gamma, const float* mean, const float* rstd,
                                       const float* dy, int64_t N, int64_t d, float* dx, float* dparams, void* ws,
                                       size_t ws_bytes, void* stream) {
  TFRS_CHECK_ARG(N >= 0 && d >= 1 && d < (1ll << 31), "layer_norm_bwd: bad shape N=%lld d=%lld", (long long)N,
                 (long long)d);
  cudaStream_t st = (cudaStream_t)stream;
  if (N == 0) {
    if (dparams) TFRS_CUDA(cudaMemsetAsync(dparams, 0, (size_t)2 * d * 4, st));
    return TFRS_OK;
  }
  TFRS_CHECK_ARG(x && mean && rstd && dy, "layer_norm_bwd: NULL pointer");
  long long chunk, parts;
  ln_chunks(N, &chunk, &parts);
  if (dparams) {
    if (!ws || ws_bytes < tfrs_layer_norm_bwd_workspace_bytes(N, d)) {
      set_error("layer_norm_bwd: workspace too small");
      return TFRS_ERR_WORKSPACE_TOO_SMALL;
    }
    TFRS_CHECK_ARG((reinterpret_cast<uintptr_t>(ws) & 15) == 0, "layer_norm_bwd: workspace must be 16-byte aligned");
  }
  if (!dx && !dparams) return TFRS_OK;
  float* part = dparams ? static_cast<float*>(ws) : nullptr;
  ln_bwd_kernel<<<(unsigned)parts, LN_THREADS, 0, st>>>(x, gamma, mean, rstd, dy, N, d, chunk, dx, part);
  TFRS_LAUNCH_CHECK();
  if (!dparams) return TFRS_OK;
  return reduce_parts(part, 1, 2 * d, (int)parts, dparams, 2 * d, st);
}
