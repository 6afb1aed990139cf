// cross_tc.cu -- K5 on the tensor cores: DCN-v2 cross layer forward (layers/feature_interaction/dcn.py:176-186)
//   out = x0 * (x . W + bias + diag_scale * x) + x        W [D,D] in Keras [in,out] layout
// as ONE wgmma GEMM with the whole cross formula in the epilogue.
//
// fp32 parity on fp16 tensor cores: each operand is rescaled by an exact power of two and split into
//   v = hi + lo,  hi = fp16(v), lo = fp16(v - hi)            (|v - hi - lo| <= 2^-22 |v|)
// and the product is accumulated in fp32 (registers) as  hi_x*hi_w + lo_x*hi_w + hi_x*lo_w  (the dropped
// lo*lo term is 2^-22 relative), i.e. 3 MMAs per K step -- ~2^-21 relative error, inside the 1e-5 bar.
//
// Layout: x (per call) and W^T (once per weight version) are turned into GMMA SWIZZLE_128B K-major tile
// images, 128 rows x 64 K-elements per 16 KB block, hi block then lo block per K slab (32 KB per slab).
// Kernel: persistent CTAs (1/SM, 544 threads) over (256-row block, 128-column tile) pairs; per K slab a
// bulk-TMA stage brings 2x(hi,lo) A blocks + (hi,lo) of W^T (96 KB); each of 4 consumer warpgroups owns 64 rows
// and issues 12 wgmma m64n128k16 (3 products x 4 K16 steps) per slab into its register accumulators, then applies
// the formula on its fragment (fetch x0 / x / bias, store fp32).  The warpgroups run independently, so one's
// MMAs overlap another's epilogue; a single producer warp (warp 16) drives the bulk-TMA ring.
#include <cuda_fp16.h>
#include "common.cuh"
#include "tc_ptx.cuh"
#include "tc_split.cuh"

namespace tfrs {
namespace tc {

constexpr int CX_THREADS = 544;
constexpr int CX_STAGES = 2;
constexpr int CX_STAGE_BYTES = 6 * 16384;  // A: 2 blocks x (hi, lo); B: (hi, lo)
struct CrossParams {
  const unsigned char* ximg;  // [n_mtiles128][kb][hi|lo][16 KB]
  const unsigned char* wimg;  // [n_ntiles128][kb][hi|lo][16 KB]   (W^T: rows = output column)
  const CxStats* xst; const CxStats* wst;
  const float* x0; const float* x; const float* bias; float diag;
  float* out; float* prod;
  long long B; int D; long long ld;
  int kb, n_mb, n_nt;
  unsigned int* out_amax;     // nullable: max |out| (float bits) accumulated by the epilogue -- the next layer's rescale statistic
};

__global__ void __launch_bounds__(CX_THREADS, 1)
cross_tc_kernel(const CrossParams p) {
  extern __shared__ __align__(1024) unsigned char cx_raw[];
  unsigned char* smem = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(cx_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + CX_STAGES * CX_STAGE_BYTES);
  uint64_t* full = bars;                  // [CX_STAGES]
  uint64_t* empty = bars + CX_STAGES;     // [CX_STAGES]

  const int wg = threadIdx.x >> 7, warp = (threadIdx.x >> 5) & 3, lane = threadIdx.x & 31;
  const long long n_tiles = (long long)p.n_mb * p.n_nt;

  if (threadIdx.x == 0) {
    for (int s = 0; s < CX_STAGES; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], 16); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (wg == 4) {
    if (threadIdx.x == 512) {
      int stage = 0; uint32_t phase = 0;
      for (long long t = blockIdx.x; t < n_tiles; t += gridDim.x) {
        const long long mb = t / p.n_nt; const int nt = (int)(t % p.n_nt);
        for (int ks = 0; ks < p.kb; ++ks) {
          mbar_wait(&empty[stage], phase ^ 1);
          mbar_expect_tx(&full[stage], CX_STAGE_BYTES);
          unsigned char* s = smem + stage * CX_STAGE_BYTES;
          bulk_g2s(s, p.ximg + ((mb * 2 + 0) * p.kb + ks) * 32768, 32768, &full[stage]);
          bulk_g2s(s + 32768, p.ximg + ((mb * 2 + 1) * p.kb + ks) * 32768, 32768, &full[stage]);
          bulk_g2s(s + 65536, p.wimg + ((long long)nt * p.kb + ks) * 32768, 32768, &full[stage]);
          if (++stage == CX_STAGES) { stage = 0; phase ^= 1; }
        }
      }
    }
    return;
  }
  // warpgroup c: rows [64 c, 64 c + 64) of the 256-row block = half (c & 1) of A block c / 2
  const int c = wg;
  const uint32_t a_off = (uint32_t)((c >> 1) * 32768 + (c & 1) * 8192);
  const float unscale = ldexpf(1.0f, -(p.xst->exp + p.wst->exp));
  float amax_out = 0.f;       // max |out| over this thread's elements (only used when p.out_amax is given)
  int stage = 0; uint32_t phase = 0;
  for (long long t = blockIdx.x; t < n_tiles; t += gridDim.x) {
    const long long mb = t / p.n_nt; const int nt = (int)(t % p.n_nt);
    float acc[64];
    for (int ks = 0; ks < p.kb; ++ks) {
      mbar_wait(&full[stage], phase);
      const uint32_t sb = smem_u32(smem + stage * CX_STAGE_BYTES);
      const uint64_t a_hi = make_smem_desc(sb + a_off), a_lo = make_smem_desc(sb + a_off + 16384);
      const uint64_t b_hi = make_smem_desc(sb + 65536), b_lo = make_smem_desc(sb + 65536 + 16384);
      wgmma_fence();
#pragma unroll
      for (int k4 = 0; k4 < 4; ++k4) {
        const uint64_t o = (uint64_t)(k4 * 2);
        wgmma_m64n128_ss(acc, a_hi + o, b_hi + o, (uint32_t)((ks | k4) != 0));
        wgmma_m64n128_ss(acc, a_lo + o, b_hi + o, 1u);
        wgmma_m64n128_ss(acc, a_hi + o, b_lo + o, 1u);
      }
      wgmma_commit();
      wgmma_wait<0>();
      acc_fence(acc);
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty[stage]);
      if (++stage == CX_STAGES) { stage = 0; phase ^= 1; }
    }
    // epilogue on the fragment: lane pairs of adjacent columns, rows r and r + 8 of the warp's 16
    const long long row_base = mb * 256 + c * 64 + warp * 16;
    const int n_base = nt * 128;
#pragma unroll
    for (int i = 0; i < 64; ++i) {
      const long long rr = row_base + frag_row(i, lane);
      const int col = n_base + frag_col(i, lane);
      if (rr < p.B && col < p.D) {
        const long long o = rr * p.ld + col;
        const float xv = __ldg(p.x + o), x0v = __ldg(p.x0 + o);
        float pv = fmaf(acc[i], unscale, p.bias ? __ldg(p.bias + col) : 0.f);
        pv = fmaf(p.diag, xv, pv);
        if (p.prod) p.prod[o] = pv;
        const float ov = fmaf(x0v, pv, xv);
        p.out[o] = ov;
        amax_out = fmaxf(amax_out, fabsf(ov));
      }
    }
  }
  if (p.out_amax) {   // same statistic, same bits, as a cx_amax_kernel pass over `out` (max is order-independent)
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) amax_out = fmaxf(amax_out, __shfl_xor_sync(0xffffffffu, amax_out, o));
    if (lane == 0 && amax_out > 0.f) atomicMax(p.out_amax, __float_as_uint(amax_out));
  }
}

}  // namespace tc
}  // namespace tfrs
using namespace tfrs;
using namespace tfrs::tc;

// ---- W image (built once per weight version, by the caller) --------------------------------------------
extern "C" size_t tfrs_cross_tc_weight_bytes(int D) {
  if (D <= 0) return 0;
  return 1024 + cx_img_bytes(D, D);
}
extern "C" int tfrs_cross_tc_weight_build(const float* W, int D, void* wbuf, size_t bytes, void* stream) {
  TFRS_CHECK_ARG(W && wbuf && D > 0, "cross_tc_weight_build: bad arguments");
  TFRS_CHECK_ARG(bytes >= tfrs_cross_tc_weight_bytes(D), "cross_tc_weight_build: buffer too small");
  TFRS_CHECK_ARG((reinterpret_cast<uintptr_t>(wbuf) & 15) == 0, "cross_tc_weight_build: buffer must be 16-byte aligned");
  cudaStream_t st = (cudaStream_t)stream;
  CxStats* ws = (CxStats*)wbuf;
  TFRS_CUDA(cudaMemsetAsync(wbuf, 0, 1024, st));
  cx_amax_kernel<<<64, 256, 0, st>>>(W, D, D, D, ws);
  TFRS_LAUNCH_CHECK();
  cx_exp_kernel<<<1, 1, 0, st>>>(ws);
  TFRS_LAUNCH_CHECK();
  const int kb = (int)ceil_div(D, 64);
  const long long nt = ceil_div(D, 128);
  const long long chunks = nt * 128 * kb * 8;
  // rows of the image = output columns n; element (n, k) = W[k, n]  -> transposed read
  cx_split_image_kernel<true><<<(unsigned)ceil_div(chunks, 256), 256, 0, st>>>(W, D, D, D, kb, nt, ws, (unsigned char*)wbuf + 1024);
  TFRS_LAUNCH_CHECK();
  return TFRS_OK;
}

extern "C" size_t tfrs_cross_tc_workspace_bytes(int64_t B, int D) {
  if (B <= 0 || D <= 0) return 0;
  return 1024 + cx_img_bytes(ceil_div(B, 256) * 256, D);
}

extern "C" int tfrs_cross_tc_fwd_ex_f32(const float* x0, const float* x, const void* wbuf, const float* bias, int64_t B, int D,
                                        int64_t ld, float diag_scale, float* out, float* prod, const unsigned int* x_amax_bits,
                                        unsigned int* out_amax_bits, void* ws, size_t ws_bytes, void* stream) {
  TFRS_CHECK_ARG(x0 && x && wbuf && out, "cross_tc_fwd: NULL pointer");
  TFRS_CHECK_ARG(B > 0 && D > 0 && ld >= D, "cross_tc_fwd: bad shape");
  TFRS_CHECK_ARG(diag_scale >= 0.f, "`diag_scale` should be non-negative. Got `diag_scale` = %g", diag_scale);
  if (!ws || ws_bytes < tfrs_cross_tc_workspace_bytes(B, D)) { set_error("cross_tc_fwd: workspace too small"); return TFRS_ERR_WORKSPACE_TOO_SMALL; }
  TFRS_CHECK_ARG((reinterpret_cast<uintptr_t>(ws) & 15) == 0, "cross_tc_fwd: workspace must be 16-byte aligned");
  cudaStream_t st = (cudaStream_t)stream;
  CxStats* xs = (CxStats*)ws;
  unsigned char* ximg = (unsigned char*)ws + 1024;
  const int kb = (int)ceil_div(D, 64);
  const int n_mb = (int)ceil_div(B, 256);
  const int n_nt = (int)ceil_div(D, 128);
  TFRS_CUDA(cudaMemsetAsync(ws, 0, 1024, st));
  if (x_amax_bits) {   // max |x| is already known (the previous layer's epilogue produced it): no pass over x
    TFRS_CUDA(cudaMemcpyAsync(&xs->amax_bits, x_amax_bits, sizeof(unsigned int), cudaMemcpyDeviceToDevice, st));
  } else {
    cx_amax_kernel<<<(unsigned)(sm_count() * 8), 256, 0, st>>>(x, B, D, ld, xs);
    TFRS_LAUNCH_CHECK();
  }
  cx_exp_kernel<<<1, 1, 0, st>>>(xs);
  TFRS_LAUNCH_CHECK();
  {
    const long long chunks = (long long)n_mb * 2 * 128 * kb * 8;
    unsigned blocks = (unsigned)(ceil_div(chunks, 256) < (1 << 20) ? ceil_div(chunks, 256) : (1 << 20));
    cx_split_image_kernel<false><<<blocks, 256, 0, st>>>(x, B, D, ld, kb, (long long)n_mb * 2, xs, ximg);
    TFRS_LAUNCH_CHECK();
  }
  if (out_amax_bits) TFRS_CUDA(cudaMemsetAsync(out_amax_bits, 0, sizeof(unsigned int), st));
  CrossParams p{};
  p.ximg = ximg; p.wimg = (const unsigned char*)wbuf + 1024; p.xst = xs; p.wst = (const CxStats*)wbuf;
  p.x0 = x0; p.x = x; p.bias = bias; p.diag = diag_scale; p.out = out; p.prod = prod;
  p.B = B; p.D = D; p.ld = ld; p.kb = kb; p.n_mb = n_mb; p.n_nt = n_nt; p.out_amax = out_amax_bits;
  const size_t smem = (size_t)CX_STAGES * CX_STAGE_BYTES + 1024 + 256;
  TFRS_DYN_SMEM(cross_tc_kernel, (int)smem);
  long long tiles = (long long)n_mb * n_nt;
  int grid = sm_count(); if (grid > tiles) grid = (int)tiles;
  cross_tc_kernel<<<grid, CX_THREADS, smem, st>>>(p);
  TFRS_LAUNCH_CHECK();
  return TFRS_OK;
}

extern "C" int tfrs_cross_tc_fwd_f32(const float* x0, const float* x, const void* wbuf, const float* bias, int64_t B, int D,
                                     int64_t ld, float diag_scale, float* out, float* prod, void* ws, size_t ws_bytes,
                                     void* stream) {
  return tfrs_cross_tc_fwd_ex_f32(x0, x, wbuf, bias, B, D, ld, diag_scale, out, prod, nullptr, nullptr, ws, ws_bytes, stream);
}
