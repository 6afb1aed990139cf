// tc_split.cuh -- exact power-of-two rescale + fp16 hi/lo split images for fp32-parity GEMMs on wgmma.
//   v = hi + lo,  hi = fp16(v), lo = fp16(v - hi)   (|v - hi - lo| <= 2^-22 |v|);  products are accumulated as
//   hi*hi + lo*hi + hi*lo in fp32 (the dropped lo*lo term is 2^-22 relative).
// Image layout: 128-row tiles x 64-wide K slabs, per slab a hi block then a lo block, each 128 rows x 128 B in
// GMMA SWIZZLE_128B K-major order (16-byte chunk j of row r at chunk j ^ (r & 7)).
#pragma once
#include <cuda_fp16.h>
#include "common.cuh"

namespace tfrs {
namespace tc {

constexpr int CX_TARGET_EXP = 14;

struct CxStats { unsigned int amax_bits; int exp; int pad0, pad1; };

// max |element| of a [rows, D] matrix with row stride ld (one warp per row: coalesced, no index division)
static __global__ void __launch_bounds__(256)
cx_amax_kernel(const float* __restrict__ src, long long rows, int D, long long ld, CxStats* __restrict__ st) {
  const int lane = threadIdx.x & 31;
  const long long warp = ((long long)blockIdx.x * 256 + threadIdx.x) >> 5;
  const long long nwarps = ((long long)gridDim.x * 256) >> 5;
  float a = 0.f;
  for (long long r = warp; r < rows; r += nwarps) {
    const float* p = src + r * ld;
    for (int c = lane; c < D; c += 32) a = fmaxf(a, fabsf(p[c]));
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) a = fmaxf(a, __shfl_xor_sync(0xffffffffu, a, o));
  __shared__ float red[8];
  if (lane == 0) red[threadIdx.x >> 5] = a;
  __syncthreads();
  if (threadIdx.x == 0) {  // one atomic per CTA (non-negative floats order like their bit patterns)
#pragma unroll
    for (int i = 1; i < 8; ++i) a = fmaxf(a, red[i]);
    if (a > 0.f) atomicMax(&st->amax_bits, __float_as_uint(a));
  }
}
// grid for cx_amax_kernel: one warp per row, capped at a few CTAs per SM (the kernel strides over the rows)
static inline unsigned cx_amax_grid(long long rows) {
  const long long want = ceil_div(rows * 32, 256), cap = (long long)sm_count() * 4;
  return (unsigned)(want < cap ? (want > 0 ? want : 1) : cap);
}
static __global__ void cx_exp_kernel(CxStats* st) {
  const float amax = __uint_as_float(st->amax_bits);
  int x = 0;
  const bool ok = amax > 0.f && amax < INFINITY;
  if (ok) (void)frexpf(amax, &x);
  st->exp = ok ? (CX_TARGET_EXP - x) : 0;
}

// fp32 [rows, K] (row stride ld) -> hi/lo fp16 tile image:
//   tile t (128 rows) : slab s (64 K) : {hi, lo} : 128 rows x 128 B, 16-byte chunk j of row r at chunk j ^ (r & 7)
static __global__ void __launch_bounds__(256)
cx_split_image_kernel(const float* __restrict__ src, long long rows, int K, long long ld, int kb, long long n_tiles,
                      const CxStats* __restrict__ st, unsigned char* __restrict__ img) {
  const int sexp = st->exp;
  const long long total = n_tiles * 128 * (long long)kb * 8;
  const unsigned int cpr = (unsigned int)(kb * 8);  // 16-byte chunks per row
  for (long long w = (long long)blockIdx.x * 256 + threadIdx.x; w < total; w += (long long)gridDim.x * 256) {
    long long row; int chunk;
    if (total < (1ll << 32)) { const unsigned int w32 = (unsigned int)w; const unsigned int r32 = w32 / cpr; row = r32; chunk = (int)(w32 - r32 * cpr); }
    else { row = w / cpr; chunk = (int)(w - row * cpr); }
    const int slab = chunk / 8, cj = chunk % 8;
    const int r = (int)(row % 128);
    const long long tile = row / 128;
    const int k0 = slab * 64 + cj * 8;
    __align__(16) __half hi[8];
    __align__(16) __half lo[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      float f = 0.f;
      if (row < rows && k0 + j < K) f = src[row * ld + k0 + j];
      const float v = ldexpf(f, sexp);
      const __half h = __float2half_rn(v);
      hi[j] = h;
      lo[j] = __float2half_rn(v - __half2float(h));
    }
    unsigned char* dst = img + (tile * kb + slab) * 32768 + r * 128 + ((cj ^ (r & 7)) * 16);
    *reinterpret_cast<uint4*>(dst) = *reinterpret_cast<const uint4*>(hi);
    *reinterpret_cast<uint4*>(dst + 16384) = *reinterpret_cast<const uint4*>(lo);
  }
}


static inline size_t cx_img_bytes(long long rows, int K) {
  return (size_t)ceil_div(rows, 128) * ceil_div(K, 64) * 32768;
}

}  // namespace tc
}  // namespace tfrs
