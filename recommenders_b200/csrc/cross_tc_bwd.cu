// cross_tc_bwd.cu -- K5b on the tensor cores: the two GEMMs of the DCN-v2 cross layer backward
//   (tape.gradient through layers/feature_interaction/dcn.py:176-186; gp = g * x0 is formed by cross.cu)
//     dx = gp . W^T + diag_scale * gp + g        [B,D] = [B,D] x [D,D]      (K = D)
//     dW = x^T . gp                              [D,D] = [D,B] x [B,D]      (K = B, the batch)
// Same fp32-parity scheme as the forward (cross_tc.cu): exact power-of-two rescale, fp16 hi/lo split of both
// operands, hi*hi + lo*hi + hi*lo accumulated in fp32 in registers (wgmma).  One kernel, two epilogues:
//   DX: A = image(gp), B = image(W) (rows = input feature, K = output feature: W as stored), formula in the epilogue.
//   DW: A = image(x^T), B = image(gp^T) built by a tiled transpose; the batch is cut into chunks of 16 K-slabs
//       (1024 rows) so an accumulation chain is as short as the forward's (the tensor core's fp32 adder
//       truncates; long chains drift), every chunk stores a partial [D,D] and a fixed-order fp32 reduction sums
//       them -- deterministic, no atomics.
// Work items (chunk, 256-row block, 128-column tile) are spread over persistent 544-thread CTAs (4 consumer warpgroups + 1 producer warp); items of the
// same chunk run concurrently so their image slabs are read from HBM once and shared through L2.
#include <cuda_fp16.h>
#include "common.cuh"
#include "tc_ptx.cuh"
#include "tc_split.cuh"
#include "cross_tc.cuh"
#include "dense.cuh"

namespace tfrs {
namespace tc {

constexpr int SG_THREADS2 = 544;
constexpr int SG_STAGES2 = 2;
constexpr int SG_STAGE_BYTES = 6 * 16384;  // A: 2 blocks x (hi, lo); B: (hi, lo)
constexpr int DW_CHUNK_SLABS = 16;         // 1024 batch rows per accumulation chain
// SG_DENSE + act: the Dense layer (K6), y = act(acc + bias); SG_DENSE + TFRS_ACT_SIGMOID also stores the logits into prod
enum { SG_DX = 1, SG_DW = 2, SG_PLAIN = 3, SG_CROSS = 4, SG_DENSE = 8 };

struct SgParams {
  const unsigned char* aimg; const unsigned char* bimg;  // [tile128][kb_total][hi|lo][16 KB]
  const CxStats* ast; const CxStats* bst;
  int kb_total, kb_chunk, n_mb, n_nt, n_kc;
  long long M, N;                     // valid rows / columns of the product
  const float* e0; long long ld0;     // DX: gp (ld D);            CROSS: x0
  const float* e1; long long ld1;     // DX: g = dout;             CROSS: x
  const float* bias;                  // CROSS: bias [N] (nullable)
  float diag;
  float* out; long long ld_out;       // DX: dx;  DW: partial [n_kc][M][N];  PLAIN: C;  CROSS: out
  float* prod;                        // CROSS: x.W + bias + diag*x for the backward pass (nullable, ld_out)
};

template <int MODE>
__global__ void __launch_bounds__(SG_THREADS2, 1)
split_gemm_kernel(const SgParams p) {
  extern __shared__ __align__(1024) unsigned char sg_raw[];
  unsigned char* smem = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(sg_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + SG_STAGES2 * SG_STAGE_BYTES);
  uint64_t* full = bars;
  uint64_t* empty = bars + SG_STAGES2;

  const int wg = threadIdx.x >> 7, warp = (threadIdx.x >> 5) & 3, lane = threadIdx.x & 31;
  const long long per_chunk = (long long)p.n_mb * p.n_nt;
  const long long n_items = per_chunk * p.n_kc;

  if (threadIdx.x == 0) {
    for (int s = 0; s < SG_STAGES2; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], 16); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (wg == 4) {
    if (threadIdx.x == 512) {
      int stage = 0; uint32_t phase = 0;
      for (long long t = blockIdx.x; t < n_items; t += gridDim.x) {
        const int kc = (int)(t / per_chunk); const long long rem = t - kc * per_chunk;
        const long long mb = rem / p.n_nt; const int nt = (int)(rem % p.n_nt);
        const int k0 = kc * p.kb_chunk, k1 = min(p.kb_total, k0 + p.kb_chunk);
        for (int ks = k0; ks < k1; ++ks) {
          mbar_wait(&empty[stage], phase ^ 1);
          mbar_expect_tx(&full[stage], SG_STAGE_BYTES);
          unsigned char* s = smem + stage * SG_STAGE_BYTES;
          bulk_g2s(s, p.aimg + ((mb * 2 + 0) * p.kb_total + ks) * 32768, 32768, &full[stage]);
          bulk_g2s(s + 32768, p.aimg + ((mb * 2 + 1) * p.kb_total + ks) * 32768, 32768, &full[stage]);
          bulk_g2s(s + 65536, p.bimg + ((long long)nt * p.kb_total + ks) * 32768, 32768, &full[stage]);
          if (++stage == SG_STAGES2) { stage = 0; phase ^= 1; }
        }
      }
    }
    return;
  }
  // warpgroup c: rows [64 c, 64 c + 64) of the 256-row block = half (c & 1) of A block c / 2
  const int c = wg;
  const uint32_t a_off = (uint32_t)((c >> 1) * 32768 + (c & 1) * 8192);
  const float unscale = ldexpf(1.0f, -(p.ast->exp + p.bst->exp));
  int stage = 0; uint32_t phase = 0;
  for (long long t = blockIdx.x; t < n_items; t += gridDim.x) {
    const int kc = (int)(t / per_chunk); const long long rem = t - kc * per_chunk;
    const long long mb = rem / p.n_nt; const int nt = (int)(rem % p.n_nt);
    const int k0 = kc * p.kb_chunk, k1 = min(p.kb_total, k0 + p.kb_chunk);
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
        wgmma_m64n128_ss(acc, a_hi + o, b_hi + o, (uint32_t)((ks != k0) | (k4 != 0)));
        wgmma_m64n128_ss(acc, a_lo + o, b_hi + o, 1u);
        wgmma_m64n128_ss(acc, a_hi + o, b_lo + o, 1u);
      }
      wgmma_commit();
      wgmma_wait<0>();
      acc_fence(acc);
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty[stage]);
      if (++stage == SG_STAGES2) { stage = 0; phase ^= 1; }
    }
    const long long row_base = mb * 256 + c * 64 + warp * 16;
    const int n_base = nt * 128;
#pragma unroll
    for (int i = 0; i < 64; ++i) {
      const long long rr = row_base + frag_row(i, lane);
      const long long col = n_base + frag_col(i, lane);
      if (rr >= p.M || col >= p.N) continue;
      if (MODE == SG_DW) {
        p.out[(long long)kc * p.M * p.N + rr * p.N + col] = acc[i] * unscale;
      } else if (MODE == SG_PLAIN) {
        p.out[rr * p.ld_out + col] = acc[i] * unscale;
      } else if (MODE == SG_CROSS) {   // out = x0 * (acc + bias + diag * x) + x   (dcn.py:176-186)
        const float x0v = __ldg(p.e0 + rr * p.ld0 + col), xv = __ldg(p.e1 + rr * p.ld1 + col);
        float pv = fmaf(acc[i], unscale, p.bias ? __ldg(p.bias + col) : 0.f);
        pv = fmaf(p.diag, xv, pv);
        if (p.prod) p.prod[rr * p.ld_out + col] = pv;
        p.out[rr * p.ld_out + col] = fmaf(x0v, pv, xv);
      } else if (MODE >= SG_DENSE) {    // DENSE: y = act(acc + bias)   (Keras Dense: MatMul, BiasAdd, activation)
        const float z = fmaf(acc[i], unscale, p.bias ? __ldg(p.bias + col) : 0.f);
        if (MODE == SG_DENSE + TFRS_ACT_SIGMOID && p.prod) p.prod[rr * p.ld_out + col] = z;
        p.out[rr * p.ld_out + col] = dense_act(MODE - SG_DENSE, z);
      } else {                          // DX: dx = acc + diag * gp + g
        float v = fmaf(acc[i], unscale, __ldg(p.e1 + rr * p.ld1 + col));
        if (p.diag != 0.f) v = fmaf(p.diag, __ldg(p.e0 + rr * p.ld0 + col), v);
        p.out[rr * p.ld_out + col] = v;
      }
    }
  }
}

// fp32 src [K, M] (row stride ld)  ->  hi/lo fp16 image of src^T: image rows = columns m of src, reduction index = rows
// k of src.  One CTA per (64-row K slab, 128-column tile): coalesced 512-byte row reads, transpose through shared
// memory, 128-byte swizzled row writes.
__global__ void __launch_bounds__(256)
cx_split_image_t_kernel(const float* __restrict__ src, long long K, int M, long long ld, int kb_total,
                        const CxStats* __restrict__ st, unsigned char* __restrict__ img) {
  __shared__ float tile[64][129];
  const int ks = blockIdx.x, mt = blockIdx.y;
  const float sc = ldexpf(1.0f, st->exp);  // exact power of two (|exp| is far inside the float range)
#pragma unroll 8
  for (int e = threadIdx.x; e < 64 * 128; e += 256) {
    const int kk = e >> 7, mm = e & 127;
    const long long k = (long long)ks * 64 + kk; const int m = mt * 128 + mm;
    const float f = (k < K && m < M) ? __ldg(src + k * ld + m) : 0.f;
    tile[kk][mm] = f * sc;
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

__global__ void __launch_bounds__(256)
sg_reduce_chunks_kernel(const float* __restrict__ partial, long long elems, int chunks, float* __restrict__ out) {
  const long long e = (long long)blockIdx.x * 256 + threadIdx.x;
  if (e >= elems) return;
  float a = partial[e];
  for (int z = 1; z < chunks; ++z) a += partial[(long long)z * elems + e];
  out[e] = a;
}

struct CbPlan {
  int n_mb_b, n_mb_d, n_nt, kb_d, kb_b, n_kc;
  size_t o_st, o_gpimg, o_wimg, o_xtimg, o_gptimg, o_partial, total;
};
static void cb_plan(long long B, int D, CbPlan& pl) {
  pl.n_mb_b = (int)ceil_div(B, 256); pl.n_mb_d = (int)ceil_div(D, 256); pl.n_nt = (int)ceil_div(D, 128);
  pl.kb_d = (int)ceil_div(D, 64); pl.kb_b = (int)ceil_div(B, 64);
  pl.n_kc = (int)ceil_div(pl.kb_b, DW_CHUNK_SLABS);
  size_t o = 0;
  auto take = [&](size_t bytes) { size_t r = o; o += align_up(bytes, 1024); return r; };
  pl.o_st = take(4 * 1024);  // CxStats of gp, W, x (one 1 KB slot each)
  pl.o_gpimg = take((size_t)pl.n_mb_b * 2 * pl.kb_d * 32768);
  pl.o_wimg = take((size_t)pl.n_nt * pl.kb_d * 32768);
  pl.o_xtimg = take((size_t)pl.n_mb_d * 2 * pl.kb_b * 32768);
  pl.o_gptimg = take((size_t)pl.n_nt * pl.kb_b * 32768);
  pl.o_partial = take((size_t)pl.n_kc * D * D * 4);
  pl.total = o;
}

size_t cross_tc_bwd_gemm_workspace(long long B, int D) {
  if (B <= 0 || D <= 0) return 0;
  CbPlan pl; cb_plan(B, D, pl);
  return pl.total;
}

static int sg_launch(int mode, const SgParams& p, cudaStream_t st) {
  const size_t smem = (size_t)SG_STAGES2 * SG_STAGE_BYTES + 1024 + 256;
  TFRS_DYN_SMEM(split_gemm_kernel<SG_DX>, (int)smem);
  TFRS_DYN_SMEM(split_gemm_kernel<SG_DW>, (int)smem);
  TFRS_DYN_SMEM(split_gemm_kernel<SG_PLAIN>, (int)smem);
  TFRS_DYN_SMEM(split_gemm_kernel<SG_CROSS>, (int)smem);
  TFRS_DYN_SMEM(split_gemm_kernel<SG_DENSE + TFRS_ACT_LINEAR>, (int)smem);
  TFRS_DYN_SMEM(split_gemm_kernel<SG_DENSE + TFRS_ACT_RELU>, (int)smem);
  TFRS_DYN_SMEM(split_gemm_kernel<SG_DENSE + TFRS_ACT_SIGMOID>, (int)smem);
  const long long items = (long long)p.n_mb * p.n_nt * p.n_kc;
  int grid = sm_count(); if (grid > items) grid = (int)items;
  if (mode == SG_DX) split_gemm_kernel<SG_DX><<<grid, SG_THREADS2, smem, st>>>(p);
  else if (mode == SG_DW) split_gemm_kernel<SG_DW><<<grid, SG_THREADS2, smem, st>>>(p);
  else if (mode == SG_PLAIN) split_gemm_kernel<SG_PLAIN><<<grid, SG_THREADS2, smem, st>>>(p);
  else if (mode == SG_DENSE + TFRS_ACT_LINEAR) split_gemm_kernel<SG_DENSE + TFRS_ACT_LINEAR><<<grid, SG_THREADS2, smem, st>>>(p);
  else if (mode == SG_DENSE + TFRS_ACT_RELU) split_gemm_kernel<SG_DENSE + TFRS_ACT_RELU><<<grid, SG_THREADS2, smem, st>>>(p);
  else if (mode == SG_DENSE + TFRS_ACT_SIGMOID) split_gemm_kernel<SG_DENSE + TFRS_ACT_SIGMOID><<<grid, SG_THREADS2, smem, st>>>(p);
  else split_gemm_kernel<SG_CROSS><<<grid, SG_THREADS2, smem, st>>>(p);
  TFRS_LAUNCH_CHECK();
  return TFRS_OK;
}

// ---- general split-fp16 GEMM: C[M,N] = A'[M,K] . B'[N,K]^T with one of the epilogues above ------------------------------
// An operand is described by where element (row r of the image, reduction index k) lives in memory.
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

// out[m*ld + n] = sum_z partial[z][m][n]  (z ascending: deterministic)
__global__ void __launch_bounds__(256)
sg_reduce_chunks_strided_kernel(const float* __restrict__ partial, long long M, long long N, int chunks, float* __restrict__ out, long long ld) {
  const long long e = (long long)blockIdx.x * 256 + threadIdx.x;
  if (e >= M * N) return;
  float a = partial[e];
  for (int z = 1; z < chunks; ++z) a += partial[(long long)z * M * N + e];
  out[(e / N) * ld + (e % N)] = a;
}

// The same fixed-order sum, then the Dense epilogue: y = act(sum + bias[n]); logits (nullable) = sum + bias[n]
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

static int gt_image(const GemmOperand& op, long long rows, long long K, int kb, long long n_tiles128, CxStats* st_, unsigned char* img,
                    cudaStream_t st) {
  // max |element|: the operand's memory is [rows, K] (ld) or, transposed, [K, rows] (ld)
  if (op.transposed) cx_amax_kernel<<<cx_amax_grid(K), 256, 0, st>>>(op.ptr, K, (int)rows, op.ld, st_);
  else cx_amax_kernel<<<cx_amax_grid(rows), 256, 0, st>>>(op.ptr, rows, (int)K, op.ld, st_);
  TFRS_LAUNCH_CHECK();
  cx_exp_kernel<<<1, 1, 0, st>>>(st_);
  TFRS_LAUNCH_CHECK();
  if (op.transposed) {   // tiled shared-memory transpose: coalesced on both sides
    cx_split_image_t_kernel<<<dim3((unsigned)kb, (unsigned)n_tiles128), 256, 0, st>>>(op.ptr, K, (int)rows, op.ld, kb, st_, img);
  } else {
    const long long chunks = n_tiles128 * 128 * (long long)kb * 8;
    const unsigned g = (unsigned)(ceil_div(chunks, 256) < (1 << 20) ? ceil_div(chunks, 256) : (1 << 20));
    cx_split_image_kernel<false><<<g, 256, 0, st>>>(op.ptr, rows, (int)K, op.ld, kb, n_tiles128, st_, img);
  }
  TFRS_LAUNCH_CHECK();
  return TFRS_OK;
}

int gemm_tc(const GemmOperand& A, const GemmOperand& Bop, long long M, long long N, long long K, const GemmEpilogue& ep,
            float* out, long long ld_out, void* ws, size_t ws_bytes, cudaStream_t st) {
  GtPlan pl; gt_plan(M, N, K, pl);
  if (!ws || ws_bytes < pl.total) { set_error("gemm_tc: workspace too small"); return TFRS_ERR_WORKSPACE_TOO_SMALL; }
  TFRS_CHECK_ARG((reinterpret_cast<uintptr_t>(ws) & 15) == 0, "gemm_tc: workspace must be 16-byte aligned");
  TFRS_CHECK_ARG(N < (1ll << 31) && M < (1ll << 31), "gemm_tc: M / N too large");
  if (ep.mode != GEMM_EPI_PLAIN && ep.mode != GEMM_EPI_DENSE && pl.n_kc > 1) { set_error("gemm_tc: fused epilogues need K <= %d", DW_CHUNK_SLABS * 64); return TFRS_ERR_UNSUPPORTED; }
  unsigned char* w8 = (unsigned char*)ws;
  CxStats* ast = (CxStats*)(w8 + pl.o_st); CxStats* bst = (CxStats*)(w8 + pl.o_st + 1024);
  TFRS_CUDA(cudaMemsetAsync(w8 + pl.o_st, 0, 2048, st));
  int rc = gt_image(A, M, K, pl.kb, (long long)pl.n_mb * 2, ast, w8 + pl.o_aimg, st);
  if (rc) return rc;
  rc = gt_image(Bop, N, K, pl.kb, pl.n_nt, bst, w8 + pl.o_bimg, st);
  if (rc) return rc;
  SgParams p{};
  p.aimg = w8 + pl.o_aimg; p.bimg = w8 + pl.o_bimg; p.ast = ast; p.bst = bst;
  p.kb_total = pl.kb; p.n_mb = pl.n_mb; p.n_nt = pl.n_nt; p.M = M; p.N = N;
  p.e0 = ep.e0; p.ld0 = ep.ld0; p.e1 = ep.e1; p.ld1 = ep.ld1; p.bias = ep.bias; p.diag = ep.diag; p.prod = ep.prod;
  if (pl.n_kc > 1) {   // long reduction (the batch): chunked accumulation chains, fixed-order sum of the partials
    p.kb_chunk = DW_CHUNK_SLABS; p.n_kc = pl.n_kc; p.out = (float*)(w8 + pl.o_partial); p.ld_out = N;
    rc = sg_launch(SG_DW, p, st);
    if (rc) return rc;
    if (ep.mode == GEMM_EPI_DENSE)   // bias + activation applied to the reduced sum
      sg_reduce_chunks_dense_kernel<<<(unsigned)ceil_div(M * N, 256), 256, 0, st>>>(p.out, M, N, pl.n_kc, ep.bias, ep.act, out, ep.prod,
                                                                                     ld_out);
    else
      sg_reduce_chunks_strided_kernel<<<(unsigned)ceil_div(M * N, 256), 256, 0, st>>>(p.out, M, N, pl.n_kc, out, ld_out);
    TFRS_LAUNCH_CHECK();
    return TFRS_OK;
  }
  p.kb_chunk = pl.kb; p.n_kc = 1; p.out = out; p.ld_out = ld_out;
  if (ep.mode == GEMM_EPI_DENSE) return sg_launch(SG_DENSE + ep.act, p, st);
  return sg_launch(ep.mode == GEMM_EPI_PLAIN ? SG_PLAIN : (ep.mode == GEMM_EPI_CROSS ? SG_CROSS : SG_DX), p, st);
}

// dx (if non-NULL) and dW (if non-NULL) from gp [B,D] (dense, ld = D), x / dout / dx with row stride ld.
// Contract with the caller: the first 4 KB of `ws` (the CxStats slots) were zeroed and slot 0's amax_bits = max |gp|.
int cross_tc_bwd_gemms(const float* x, const float* W, const float* gp, const float* dout, long long B, int D, long long ld,
                       float diag, float* dx, float* dW, void* ws, size_t ws_bytes, cudaStream_t st) {
  CbPlan pl; cb_plan(B, D, pl);
  if (!ws || ws_bytes < pl.total) { set_error("cross_tc_bwd: workspace too small"); return TFRS_ERR_WORKSPACE_TOO_SMALL; }
  TFRS_CHECK_ARG((reinterpret_cast<uintptr_t>(ws) & 15) == 0, "cross_tc_bwd: workspace must be 16-byte aligned");
  unsigned char* w8 = (unsigned char*)ws;
  CxStats* gst = (CxStats*)(w8 + pl.o_st); CxStats* wst = (CxStats*)(w8 + pl.o_st + 1024); CxStats* xst = (CxStats*)(w8 + pl.o_st + 2048);
  // gst->amax_bits was filled by the caller's element-wise pass (cross.cu: cross_bwd_elem), the other slots are zero
  cx_exp_kernel<<<1, 1, 0, st>>>(gst);
  TFRS_LAUNCH_CHECK();
  if (dx) {
    cx_amax_kernel<<<cx_amax_grid(D), 256, 0, st>>>(W, D, D, D, wst);
    TFRS_LAUNCH_CHECK();
    cx_exp_kernel<<<1, 1, 0, st>>>(wst);
    TFRS_LAUNCH_CHECK();
    const long long ca = (long long)pl.n_mb_b * 2 * 128 * pl.kb_d * 8, cb = (long long)pl.n_nt * 128 * pl.kb_d * 8;
    const unsigned ga = (unsigned)(ceil_div(ca, 256) < (1 << 20) ? ceil_div(ca, 256) : (1 << 20));
    cx_split_image_kernel<false><<<ga, 256, 0, st>>>(gp, B, D, D, pl.kb_d, (long long)pl.n_mb_b * 2, gst, w8 + pl.o_gpimg);
    TFRS_LAUNCH_CHECK();
    // B operand rows = input feature i, K = output feature o: element (i, o) = W[i, o]  -> W as stored
    cx_split_image_kernel<false><<<(unsigned)ceil_div(cb, 256), 256, 0, st>>>(W, D, D, D, pl.kb_d, pl.n_nt, wst, w8 + pl.o_wimg);
    TFRS_LAUNCH_CHECK();
    SgParams p{};
    p.aimg = w8 + pl.o_gpimg; p.bimg = w8 + pl.o_wimg; p.ast = gst; p.bst = wst;
    p.kb_total = pl.kb_d; p.kb_chunk = pl.kb_d; p.n_mb = pl.n_mb_b; p.n_nt = pl.n_nt; p.n_kc = 1;
    p.M = B; p.N = D; p.e0 = gp; p.ld0 = D; p.e1 = dout; p.ld1 = ld; p.diag = diag; p.out = dx; p.ld_out = ld;
    int rc = sg_launch(SG_DX, p, st);
    if (rc) return rc;
  }
  if (dW) {
    cx_amax_kernel<<<cx_amax_grid(B), 256, 0, st>>>(x, B, D, ld, xst);
    TFRS_LAUNCH_CHECK();
    cx_exp_kernel<<<1, 1, 0, st>>>(xst);
    TFRS_LAUNCH_CHECK();
    cx_split_image_t_kernel<<<dim3((unsigned)pl.kb_b, (unsigned)(pl.n_mb_d * 2)), 256, 0, st>>>(x, B, D, ld, pl.kb_b, xst, w8 + pl.o_xtimg);
    TFRS_LAUNCH_CHECK();
    cx_split_image_t_kernel<<<dim3((unsigned)pl.kb_b, (unsigned)pl.n_nt), 256, 0, st>>>(gp, B, D, D, pl.kb_b, gst, w8 + pl.o_gptimg);
    TFRS_LAUNCH_CHECK();
    float* partial = (float*)(w8 + pl.o_partial);
    SgParams p{};
    p.aimg = w8 + pl.o_xtimg; p.bimg = w8 + pl.o_gptimg; p.ast = xst; p.bst = gst;
    p.kb_total = pl.kb_b; p.kb_chunk = DW_CHUNK_SLABS; p.n_mb = pl.n_mb_d; p.n_nt = pl.n_nt; p.n_kc = pl.n_kc;
    p.M = D; p.N = D; p.out = partial; p.ld_out = D;
    int rc = sg_launch(SG_DW, p, st);
    if (rc) return rc;
    sg_reduce_chunks_kernel<<<(unsigned)ceil_div((long long)D * D, 256), 256, 0, st>>>(partial, (long long)D * D, pl.n_kc, dW);
    TFRS_LAUNCH_CHECK();
  }
  return TFRS_OK;
}

}  // namespace tc
}  // namespace tfrs
