// split_gemm.cu -- the split-fp16 tensor-core GEMM:  C[M,N] = A'[M,K] . B'[N,K]^T  with a fused epilogue.  It runs the
// full-rank and low-rank Cross layers (K5, forward and backward), the Dense layer (K6) and tfrs_gemm_tc_f32.
//
// fp32 parity on fp16 tensor cores: each operand is rescaled by an exact power of two and split into
//   v = hi + lo,  hi = fp16(v), lo = fp16(v - hi)            (|v - hi - lo| <= 2^-22 |v|)
// and the product is accumulated in fp32 (registers) as  hi_a*hi_b + lo_a*hi_b + hi_a*lo_b  (the dropped lo*lo term is
// 2^-22 relative), i.e. 3 MMAs per K16 step -- ~2^-21 relative error, inside the 1e-5 bar.
//
// Both operands are turned into GMMA SWIZZLE_128B K-major tile images (tc_split.cuh; a transposed operand through a tiled
// shared-memory transpose).  Persistent CTAs (1/SM, 544 threads) walk (256-row block, 128-column tile) items; per 64-wide
// K slab a bulk-TMA stage brings 2x(hi,lo) A blocks + (hi,lo) B blocks (96 KB, 2 stages); each of 4 consumer warpgroups
// owns 64 rows and issues 12 wgmma m64n128k16 per slab into its register accumulators, then applies the epilogue on its
// fragment.  The warpgroups run independently, so one's MMAs overlap another's epilogue; warp 16 drives the TMA ring.
// Long reductions (K > 1024: the batch of a weight gradient, a Cross layer wider than 1024) are cut into chunks of 16
// K slabs (the tensor core's fp32 adder truncates; long chains drift); every chunk stores a partial [M,N] (mode DW) and
// a fixed-order fp32 reduction sums them and applies the epilogue -- deterministic, no atomics.  Items of one chunk run concurrently, so their
// image slabs are read from HBM once and shared through L2.
// Each operand's exponent puts its largest FINITE |element| in [2^13, 2^14) (finite_abs); the epilogue undoes both
// exponents exactly, also when 2^-(exp_a + exp_b) is not a normal float.
#include <cuda_fp16.h>
#include "common.cuh"
#include "tc_ptx.cuh"
#include "tc_split.cuh"
#include "split_gemm.cuh"
#include "dense.cuh"

namespace tfrs {
namespace tc {

constexpr int SG_THREADS = 544;
constexpr int SG_STAGES = 2;
constexpr int SG_STAGE_BYTES = 6 * 16384;  // A: 2 blocks x (hi, lo); B: (hi, lo)
constexpr int DW_CHUNK_SLABS = 16;         // 1024 reduction indices per accumulation chain of a chunked GEMM
// SG_DENSE + act: the Dense layer (K6), y = act(acc + bias); SG_DENSE + TFRS_ACT_SIGMOID also stores the logits into prod
enum { SG_DX = 1, SG_DW = 2, SG_PLAIN = 3, SG_CROSS = 4, SG_DENSE = 8 };

struct SgParams {
  const unsigned char* aimg; const unsigned char* bimg;  // [tile128][kb_total][hi|lo][16 KB]
  const CxStats* ast; const CxStats* bst;
  int kb_total, n_mb, n_nt, n_kc;     // n_kc: DW only, chunks of DW_CHUNK_SLABS slabs
  long long M, N;                     // valid rows / columns of the product
  const float* e0; long long ld0;     // DX: gp;       CROSS: x0 (ld_out)
  const float* e1; long long ld1;     // DX: g = dout; CROSS: x (ld_out)
  const float* bias;                  // CROSS, DENSE: bias [N] (nullable)
  float diag;
  float* out; long long ld_out;       // DW: partial [n_kc][M][N]
  float* prod;                        // CROSS: acc + bias + diag*x for the backward pass; DENSE sigmoid: logits (nullable)
  unsigned int* out_amax;             // CROSS: max |out| as float bits (nullable)
};

template <int MODE>
__global__ void __launch_bounds__(SG_THREADS, 1)
split_gemm_kernel(const SgParams p) {
  extern __shared__ __align__(1024) unsigned char sg_raw[];
  unsigned char* smem = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(sg_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + SG_STAGES * SG_STAGE_BYTES);
  uint64_t* full = bars;
  uint64_t* empty = bars + SG_STAGES;

  const int wg = threadIdx.x >> 7, warp = (threadIdx.x >> 5) & 3, lane = threadIdx.x & 31;
  const long long per_chunk = (long long)p.n_mb * p.n_nt;
  const long long n_items = MODE == SG_DW ? per_chunk * p.n_kc : per_chunk;

  if (threadIdx.x == 0) {
    for (int s = 0; s < SG_STAGES; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], 16); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (wg == 4) {
    if (threadIdx.x == 512) {
      int stage = 0; uint32_t phase = 0;
      for (long long t = blockIdx.x; t < n_items; t += gridDim.x) {
        int kc = 0; long long rem = t;
        if (MODE == SG_DW) { kc = (int)(t / per_chunk); rem = t - kc * per_chunk; }
        const long long mb = rem / p.n_nt; const int nt = (int)(rem % p.n_nt);
        const int k0 = kc * DW_CHUNK_SLABS, k1 = MODE == SG_DW ? min(p.kb_total, k0 + DW_CHUNK_SLABS) : p.kb_total;
        for (int ks = k0; ks < k1; ++ks) {
          mbar_wait(&empty[stage], phase ^ 1);
          mbar_expect_tx(&full[stage], SG_STAGE_BYTES);
          unsigned char* s = smem + stage * SG_STAGE_BYTES;
          bulk_g2s(s, p.aimg + ((mb * 2 + 0) * p.kb_total + ks) * 32768, 32768, &full[stage]);
          bulk_g2s(s + 32768, p.aimg + ((mb * 2 + 1) * p.kb_total + ks) * 32768, 32768, &full[stage]);
          bulk_g2s(s + 65536, p.bimg + ((long long)nt * p.kb_total + ks) * 32768, 32768, &full[stage]);
          if (++stage == SG_STAGES) { stage = 0; phase ^= 1; }
        }
      }
    }
    return;
  }
  // warpgroup c: rows [64 c, 64 c + 64) of the 256-row block = half (c & 1) of A block c / 2
  const int c = wg;
  const uint32_t a_off = (uint32_t)((c >> 1) * 32768 + (c & 1) * 8192);
  // the product is acc * 2^-S, S = exp_a + exp_b.  When 2^-S is not a normal float (S outside [-127, 126]: tiny or huge
  // operands whose product is still an fp32 number) that factor would round to 0 or Inf, so unscale = 0 marks the case: the
  // accumulator is scaled by ldexpf and the epilogue multiplies by 1.  Uniform across the CTA; where 2^-S is normal the bits
  // are those of acc * 2^-S.
  const int S = p.ast->exp + p.bst->exp;
  const float unscale = S >= -127 && S <= 126 ? ldexpf(1.0f, -S) : 0.f;
  float amax_out = 0.f;       // CROSS: max |out| over this thread's finite elements
  int stage = 0; uint32_t phase = 0;
  for (long long t = blockIdx.x; t < n_items; t += gridDim.x) {
    int kc = 0; long long rem = t;
    if (MODE == SG_DW) { kc = (int)(t / per_chunk); rem = t - kc * per_chunk; }
    const long long mb = rem / p.n_nt; const int nt = (int)(rem % p.n_nt);
    const int k0 = kc * DW_CHUNK_SLABS, k1 = MODE == SG_DW ? min(p.kb_total, k0 + DW_CHUNK_SLABS) : p.kb_total;
    float acc[64];
    for (int ks = k0; ks < k1; ++ks) {
      mbar_wait(&full[stage], phase);
      const uint32_t sb = smem_u32(smem + stage * SG_STAGE_BYTES);
      const uint64_t a_hi = make_smem_desc(sb + a_off), a_lo = make_smem_desc(sb + a_off + 16384);
      const uint64_t b_hi = make_smem_desc(sb + 65536), b_lo = make_smem_desc(sb + 65536 + 16384);
      wgmma_fence();
#pragma unroll
      for (int k4 = 0; k4 < 4; ++k4) {
        const uint64_t o = (uint64_t)(k4 * 2);
        wgmma_m64n128_ss(acc, a_hi + o, b_hi + o, (uint32_t)(((ks - k0) | k4) != 0));
        wgmma_m64n128_ss(acc, a_lo + o, b_hi + o, 1u);
        wgmma_m64n128_ss(acc, a_hi + o, b_lo + o, 1u);
      }
      wgmma_commit();
      wgmma_wait<0>();
      acc_fence(acc);
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty[stage]);
      if (++stage == SG_STAGES) { stage = 0; phase ^= 1; }
    }
    float u = unscale;
    if (u == 0.f) {
      const int s = p.ast->exp + p.bst->exp;
#pragma unroll
      for (int i = 0; i < 64; ++i) acc[i] = ldexpf(acc[i], -s);
      u = 1.f;
    }
    // epilogue on the fragment: lane pairs of adjacent columns, rows r and r + 8 of the warp's 16
    const long long row_base = mb * 256 + c * 64 + warp * 16;
    const int n_base = nt * 128, n_cols = (int)p.N;
#pragma unroll
    for (int i = 0; i < 64; ++i) {
      const long long rr = row_base + frag_row(i, lane);
      const int col = n_base + frag_col(i, lane);
      if (rr >= p.M || col >= n_cols) continue;
      if (MODE == SG_DW) {
        p.out[(long long)kc * p.M * p.N + rr * p.N + col] = acc[i] * u;
      } else if (MODE == SG_PLAIN) {
        p.out[rr * p.ld_out + col] = acc[i] * u;
      } else if (MODE == SG_CROSS) {   // out = x0 * (acc + bias + diag * x) + x   (dcn.py:176-186)
        const long long o = rr * p.ld_out + col;
        const float xv = __ldg(p.e1 + o), x0v = __ldg(p.e0 + o);
        float pv = fmaf(acc[i], u, p.bias ? __ldg(p.bias + col) : 0.f);
        pv = fmaf(p.diag, xv, pv);
        if (p.prod) p.prod[o] = pv;
        const float ov = fmaf(x0v, pv, xv);
        p.out[o] = ov;
        amax_out = fmaxf(amax_out, finite_abs(ov));
      } else if (MODE >= SG_DENSE) {    // DENSE: y = act(acc + bias)   (Keras Dense: MatMul, BiasAdd, activation)
        const float z = fmaf(acc[i], u, p.bias ? __ldg(p.bias + col) : 0.f);
        if (MODE == SG_DENSE + TFRS_ACT_SIGMOID && p.prod) p.prod[rr * p.ld_out + col] = z;
        p.out[rr * p.ld_out + col] = dense_act(MODE - SG_DENSE, z);
      } else {                          // DX: dx = acc + diag * gp + g
        float v = fmaf(acc[i], u, __ldg(p.e1 + rr * p.ld1 + col));
        if (p.diag != 0.f) v = fmaf(p.diag, __ldg(p.e0 + rr * p.ld0 + col), v);
        p.out[rr * p.ld_out + col] = v;
      }
    }
  }
  if (MODE == SG_CROSS && p.out_amax) {   // same bits as a cx_amax_kernel pass over `out` (max is order-independent)
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) amax_out = fmaxf(amax_out, __shfl_xor_sync(0xffffffffu, amax_out, o));
    if (lane == 0 && amax_out > 0.f) atomicMax(p.out_amax, __float_as_uint(amax_out));
  }
}

static int sg_launch(int mode, const SgParams& p, cudaStream_t st) {
  const size_t smem = (size_t)SG_STAGES * SG_STAGE_BYTES + 1024 + 256;
  TFRS_DYN_SMEM(split_gemm_kernel<SG_DX>, (int)smem);
  TFRS_DYN_SMEM(split_gemm_kernel<SG_DW>, (int)smem);
  TFRS_DYN_SMEM(split_gemm_kernel<SG_PLAIN>, (int)smem);
  TFRS_DYN_SMEM(split_gemm_kernel<SG_CROSS>, (int)smem);
  TFRS_DYN_SMEM(split_gemm_kernel<SG_DENSE + TFRS_ACT_LINEAR>, (int)smem);
  TFRS_DYN_SMEM(split_gemm_kernel<SG_DENSE + TFRS_ACT_RELU>, (int)smem);
  TFRS_DYN_SMEM(split_gemm_kernel<SG_DENSE + TFRS_ACT_SIGMOID>, (int)smem);
  const long long items = (long long)p.n_mb * p.n_nt * (mode == SG_DW ? p.n_kc : 1);
  int grid = sm_count(); if (grid > items) grid = (int)items;
  if (mode == SG_DX) split_gemm_kernel<SG_DX><<<grid, SG_THREADS, smem, st>>>(p);
  else if (mode == SG_DW) split_gemm_kernel<SG_DW><<<grid, SG_THREADS, smem, st>>>(p);
  else if (mode == SG_PLAIN) split_gemm_kernel<SG_PLAIN><<<grid, SG_THREADS, smem, st>>>(p);
  else if (mode == SG_DENSE + TFRS_ACT_LINEAR) split_gemm_kernel<SG_DENSE + TFRS_ACT_LINEAR><<<grid, SG_THREADS, smem, st>>>(p);
  else if (mode == SG_DENSE + TFRS_ACT_RELU) split_gemm_kernel<SG_DENSE + TFRS_ACT_RELU><<<grid, SG_THREADS, smem, st>>>(p);
  else if (mode == SG_DENSE + TFRS_ACT_SIGMOID) split_gemm_kernel<SG_DENSE + TFRS_ACT_SIGMOID><<<grid, SG_THREADS, smem, st>>>(p);
  else split_gemm_kernel<SG_CROSS><<<grid, SG_THREADS, smem, st>>>(p);
  TFRS_LAUNCH_CHECK();
  return TFRS_OK;
}

// ---- the driver: operand images, then one launch (plus the partials' reduction when chunked) ------------------------------
struct GtPlan { int n_mb, n_nt, kb, n_kc; size_t o_st, o_aimg, o_bimg, o_partial, total; };
static void gt_plan(long long M, long long N, long long K, GtPlan& pl) {
  pl.n_mb = (int)ceil_div(M, 256); pl.n_nt = (int)ceil_div(N, 128); pl.kb = (int)ceil_div(K, 64);
  pl.n_kc = (int)ceil_div(pl.kb, DW_CHUNK_SLABS);
  size_t o = 0;
  auto take = [&](size_t bytes) { size_t r = o; o += align_up(bytes, 1024); return r; };
  pl.o_st = take(2048);
  pl.o_aimg = take((size_t)pl.n_mb * 2 * pl.kb * 32768);
  pl.o_bimg = take((size_t)pl.n_nt * pl.kb * 32768);
  pl.o_partial = take(pl.n_kc > 1 ? (size_t)pl.n_kc * M * N * 4 : 0);
  pl.total = o;
}
size_t gemm_tc_workspace(long long M, long long N, long long K) {
  if (M <= 0 || N <= 0 || K <= 0) return 0;
  GtPlan pl; gt_plan(M, N, K, pl);
  return pl.total;
}

// The fixed-order sum of the chunk partials (as reduce_parts), then the Dense epilogue: y = act(sum + bias[n]); logits (nullable) = sum + bias[n]
__global__ void __launch_bounds__(256)
sg_reduce_chunks_dense_kernel(const float* __restrict__ partial, long long M, long long N, int chunks, const float* __restrict__ bias,
                              int act, float* __restrict__ out, float* __restrict__ logits, long long ld) {
  const long long e = (long long)blockIdx.x * 256 + threadIdx.x;
  if (e >= M * N) return;
  float a = partial[e];
  for (int z = 1; z < chunks; ++z) a += partial[(long long)z * M * N + e];
  const long long n = e % N, o = (e / N) * ld + n;
  const float zv = bias ? a + bias[n] : a;
  if (logits) logits[o] = zv;
  out[o] = dense_act(act, zv);
}

// The fixed-order sum of the chunk partials (as reduce_parts), then the CROSS or DX epilogue of split_gemm_kernel on the sum
// (the partials are already unscaled):  CROSS: pv = sum + bias[n] + diag * x; prod = pv; out = x0 * pv + x; out_amax = max
// finite |out| (one atomic per warp: the bits of a cx_amax_kernel pass over out).  DX: out = sum + g + diag * gp.
__global__ void __launch_bounds__(256)
sg_reduce_chunks_cross_dx_kernel(const float* __restrict__ partial, long long M, long long N, int chunks, bool cross,
                                 const float* __restrict__ e0, long long ld0, const float* __restrict__ e1, long long ld1,
                                 const float* __restrict__ bias, float diag, float* __restrict__ prod, float* __restrict__ out,
                                 long long ld, unsigned int* __restrict__ out_amax) {
  const long long e = (long long)blockIdx.x * 256 + threadIdx.x;
  float amax = 0.f;
  if (e < M * N) {
    float a = partial[e];
    for (int z = 1; z < chunks; ++z) a += partial[(long long)z * M * N + e];
    const long long m = e / N, n = e % N;
    if (cross) {   // ld0 == ld1 == ld
      const long long o = m * ld + n;
      const float xv = e1[o];
      float pv = a + (bias ? bias[n] : 0.f);
      pv = fmaf(diag, xv, pv);
      if (prod) prod[o] = pv;
      const float ov = fmaf(e0[o], pv, xv);
      out[o] = ov;
      amax = finite_abs(ov);
    } else {
      float v = a + e1[m * ld1 + n];
      if (diag != 0.f) v = fmaf(diag, e0[m * ld0 + n], v);
      out[m * ld + n] = v;
    }
  }
  if (cross && out_amax) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));
    if ((threadIdx.x & 31) == 0 && amax > 0.f) atomicMax(out_amax, __float_as_uint(amax));
  }
}

int gemm_tc(const GemmOperand& A, const GemmOperand& Bop, long long M, long long N, long long K, const GemmEpilogue& ep,
            float* out, long long ld_out, void* ws, size_t ws_bytes, cudaStream_t st) {
  GtPlan pl; gt_plan(M, N, K, pl);
  if (!ws || ws_bytes < pl.total) { set_error("gemm_tc: workspace too small"); return TFRS_ERR_WORKSPACE_TOO_SMALL; }
  TFRS_CHECK_ARG((reinterpret_cast<uintptr_t>(ws) & 15) == 0, "gemm_tc: workspace must be 16-byte aligned");
  TFRS_CHECK_ARG(N < (1ll << 31) && M < (1ll << 31), "gemm_tc: M / N too large");
  TFRS_CHECK_ARG(ep.mode != GEMM_EPI_CROSS || (ep.ld0 == ld_out && ep.ld1 == ld_out), "gemm_tc: CROSS needs x0, x and out of one row stride");
  unsigned char* w8 = (unsigned char*)ws;
  CxStats* ast = (CxStats*)(w8 + pl.o_st); CxStats* bst = (CxStats*)(w8 + pl.o_st + 1024);
  TFRS_CUDA(cudaMemsetAsync(w8 + pl.o_st, 0, 2048, st));
  int rc = split_image(A.ptr, A.ld, A.transposed, A.amax_bits, M, K, pl.kb, (long long)pl.n_mb * 2, ast, w8 + pl.o_aimg, st);
  if (rc) return rc;
  rc = split_image(Bop.ptr, Bop.ld, Bop.transposed, Bop.amax_bits, N, K, pl.kb, pl.n_nt, bst, w8 + pl.o_bimg, st);
  if (rc) return rc;
  SgParams p{};
  p.aimg = w8 + pl.o_aimg; p.bimg = w8 + pl.o_bimg; p.ast = ast; p.bst = bst;
  p.kb_total = pl.kb; p.n_mb = pl.n_mb; p.n_nt = pl.n_nt; p.n_kc = pl.n_kc; p.M = M; p.N = N;
  p.e0 = ep.e0; p.ld0 = ep.ld0; p.e1 = ep.e1; p.ld1 = ep.ld1; p.bias = ep.bias; p.diag = ep.diag; p.prod = ep.prod;
  if (ep.mode == GEMM_EPI_CROSS && ep.out_amax) TFRS_CUDA(cudaMemsetAsync(ep.out_amax, 0, sizeof(unsigned int), st));
  if (pl.n_kc > 1) {   // long reduction: chunked accumulation chains, fixed-order sum of the partials, then the epilogue
    p.out = (float*)(w8 + pl.o_partial); p.ld_out = N;
    rc = sg_launch(SG_DW, p, st);
    if (rc) return rc;
    if (ep.mode == GEMM_EPI_PLAIN) return reduce_parts(p.out, M, N, pl.n_kc, out, ld_out, st);
    const unsigned grid = (unsigned)ceil_div(M * N, 256);
    if (ep.mode == GEMM_EPI_DENSE)   // bias + activation applied to the reduced sum
      sg_reduce_chunks_dense_kernel<<<grid, 256, 0, st>>>(p.out, M, N, pl.n_kc, ep.bias, ep.act, out, ep.prod, ld_out);
    else
      sg_reduce_chunks_cross_dx_kernel<<<grid, 256, 0, st>>>(p.out, M, N, pl.n_kc, ep.mode == GEMM_EPI_CROSS, ep.e0, ep.ld0, ep.e1,
                                                             ep.ld1, ep.bias, ep.diag, ep.prod, out, ld_out, ep.out_amax);
    TFRS_LAUNCH_CHECK();
    return TFRS_OK;
  }
  p.out = out; p.ld_out = ld_out;
  if (ep.mode == GEMM_EPI_DENSE) return sg_launch(SG_DENSE + ep.act, p, st);
  if (ep.mode == GEMM_EPI_CROSS) {
    p.out_amax = ep.out_amax;
    return sg_launch(SG_CROSS, p, st);
  }
  return sg_launch(ep.mode == GEMM_EPI_PLAIN ? SG_PLAIN : SG_DX, p, st);
}

}  // namespace tc
}  // namespace tfrs
