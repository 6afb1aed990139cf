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

// max |element| over the FINITE elements of a [rows, D] matrix with row stride ld (one warp per row: coalesced, no index
// division).  Inf and NaN are left out (finite_abs): the rescale then fits the finite data, and a non-finite element spoils
// only the products of its own row or column (its hi is Inf or NaN, its lo NaN), as it would in fp32.
static __global__ void __launch_bounds__(256)
cx_amax_kernel(const float* __restrict__ src, long long rows, int D, long long ld, CxStats* __restrict__ st) {
  const int lane = threadIdx.x & 31;
  const long long warp = ((long long)blockIdx.x * 256 + threadIdx.x) >> 5;
  const long long nwarps = ((long long)gridDim.x * 256) >> 5;
  float a = 0.f;
  for (long long r = warp; r < rows; r += nwarps) {
    const float* p = src + r * ld;
    for (int c = lane; c < D; c += 32) a = fmaxf(a, finite_abs(p[c]));
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

// Where an image's elements come from: element (i, j) of an fp32 matrix, at(i, j) as a plain load and at_ldg(i, j) through
// the read-only path.  MatrixSrc is a stored row-major matrix with row stride ld; split_gemm.cuh's WindowSrc is the im2col
// matrix of a 1-D convolution, gathered from its input.
struct MatrixSrc {
  const float* p; long long ld;
  __device__ __forceinline__ float at(long long i, long long j) const { return p[i * ld + j]; }
  __device__ __forceinline__ float at_ldg(long long i, long long j) const { return __ldg(p + i * ld + j); }
};

// fp32 [rows, K] -> hi/lo fp16 tile image:
//   tile t (128 rows) : slab s (64 K) : {hi, lo} : 128 rows x 128 B, 16-byte chunk j of row r at chunk j ^ (r & 7)
template <class Src>
__device__ __forceinline__ void split_image_rows(const Src& src, long long rows, int K, int kb, long long n_tiles,
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
      if (row < rows && k0 + j < K) f = src.at(row, k0 + j);
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
static __global__ void __launch_bounds__(256)
cx_split_image_kernel(const float* __restrict__ src, long long rows, int K, long long ld, int kb, long long n_tiles,
                      const CxStats* __restrict__ st, unsigned char* __restrict__ img) {
  split_image_rows(MatrixSrc{src, ld}, rows, K, kb, n_tiles, st, img);
}
// fp32 src [K, M]  ->  hi/lo fp16 image of src^T: image rows = columns m of src, reduction index = rows k of src.  One
// CTA per (64-row K slab, 128-column tile): coalesced 512-byte row reads, transpose through shared memory, 128-byte
// swizzled row writes.
template <class Src>
__device__ __forceinline__ void split_image_cols(const Src& src, long long K, int M, int kb_total, const CxStats* __restrict__ st,
                                                 unsigned char* __restrict__ img) {
  __shared__ float tile[64][129];
  const int ks = blockIdx.x, mt = blockIdx.y;
  // v * 2^exp as two exact power-of-two factors: 2^exp alone overflows when exp > 127 (max |element| < 2^-113), and exp >= -114
  // keeps 2^exp normal, so this equals ldexpf(v, exp) -- at the price of a multiply, where ldexpf per element slows the load loop
  const int e1 = min(st->exp, 127);
  const float sc1 = ldexpf(1.0f, e1), sc2 = ldexpf(1.0f, st->exp - e1);
#pragma unroll 8
  for (int e = threadIdx.x; e < 64 * 128; e += 256) {
    const int kk = e >> 7, mm = e & 127;
    const long long k = (long long)ks * 64 + kk; const int m = mt * 128 + mm;
    const float f = (k < K && m < M) ? src.at_ldg(k, m) : 0.f;
    tile[kk][mm] = f * sc1 * sc2;
  }
  __syncthreads();
  unsigned char* base = img + ((long long)mt * kb_total + ks) * 32768;
#pragma unroll
  for (int pass = 0; pass < 4; ++pass) {
    const int r = pass * 32 + (threadIdx.x >> 3), cj = threadIdx.x & 7;
    __align__(16) __half hi[8];
    __align__(16) __half lo[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float v = tile[cj * 8 + j][r];
      const __half h = __float2half_rn(v);
      hi[j] = h;
      lo[j] = __float2half_rn(v - __half2float(h));
    }
    unsigned char* dst = base + r * 128 + ((cj ^ (r & 7)) * 16);
    *reinterpret_cast<uint4*>(dst) = *reinterpret_cast<const uint4*>(hi);
    *reinterpret_cast<uint4*>(dst + 16384) = *reinterpret_cast<const uint4*>(lo);
  }
}
static __global__ void __launch_bounds__(256)
cx_split_image_t_kernel(const float* __restrict__ src, long long K, int M, long long ld, int kb_total,
                        const CxStats* __restrict__ st, unsigned char* __restrict__ img) {
  split_image_cols(MatrixSrc{src, ld}, K, M, kb_total, st, img);
}
// The split image of one operand, three launches: max |element| into st (a pass over the operand, or a copy of the caller's
// amax_bits when it already knows it), the exponent, then the hi/lo image of n_tiles 128-row tiles x kb K slabs.
// Element (image row r, reduction index k) = transposed ? src[k * ld + r] : src[r * ld + k], for r < rows and k < K; the
// rest of the image is zero.  st->amax_bits must be 0 on entry.
static inline int split_image(const float* src, long long ld, bool transposed, const unsigned int* amax_bits, long long rows,
                              long long K, int kb, long long n_tiles, CxStats* st, unsigned char* img, cudaStream_t s) {
  if (amax_bits) TFRS_CUDA(cudaMemcpyAsync(&st->amax_bits, amax_bits, sizeof(unsigned int), cudaMemcpyDeviceToDevice, s));
  else if (transposed) cx_amax_kernel<<<cx_amax_grid(K), 256, 0, s>>>(src, K, (int)rows, ld, st);
  else cx_amax_kernel<<<cx_amax_grid(rows), 256, 0, s>>>(src, rows, (int)K, ld, st);
  TFRS_LAUNCH_CHECK();
  cx_exp_kernel<<<1, 1, 0, s>>>(st);
  TFRS_LAUNCH_CHECK();
  if (transposed) {   // tiled shared-memory transpose: coalesced on both sides
    cx_split_image_t_kernel<<<dim3((unsigned)kb, (unsigned)n_tiles), 256, 0, s>>>(src, K, (int)rows, ld, kb, st, img);
  } else {
    const long long chunks = n_tiles * 128 * (long long)kb * 8;
    const unsigned g = (unsigned)(ceil_div(chunks, 256) < (1 << 20) ? ceil_div(chunks, 256) : (1 << 20));
    cx_split_image_kernel<<<g, 256, 0, s>>>(src, rows, (int)K, ld, kb, n_tiles, st, img);
  }
  TFRS_LAUNCH_CHECK();
  return TFRS_OK;
}

static inline size_t cx_img_bytes(long long rows, int K) {
  return (size_t)ceil_div(rows, 128) * ceil_div(K, 64) * 32768;
}

// How many parts to cut the streamed tiles of a (stationary block, streamed tiles) kernel into, so that n_blocks x parts CTAs
// fill the GPU: minimise waves x (tiles per CTA + ~6 tile times of fixed cost: stationary load, pipeline fill and drain,
// epilogue, partials).
static inline int stream_parts(long long n_blocks, long long n_tiles) {
  int parts = 1; double best = 1e30;
  const int sms = sm_count();
  for (int c = 1; c <= 16 && c <= n_tiles; ++c) {
    const double cost = (double)ceil_div(n_blocks * c, sms) * ((double)ceil_div(n_tiles, c) + 6.0);
    if (cost < best * 0.97) { best = cost; parts = c; }
  }
  return parts;
}

}  // namespace tc
}  // namespace tfrs
