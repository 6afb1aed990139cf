// softmax_tc_bwd.cu -- K3b on the tensor cores: backward of the in-batch softmax loss of tfrs.tasks.Retrieval
//   (tape.gradient at models/base.py:77 through tasks/retrieval.py:178-210)
//   G_ij = (softmax(s)_ij - [i == j]) * w_i * grad_loss / T ;   dq = G . c  [B,d] ;   dc = G^T . q  [C,d]
// as two launches of ONE kernel (flash-attention-backward shape, deterministic -- no atomics):
//   stationary operand X (128 rows, resident in smem), streaming operand Y (128-row tiles, bulk-TMA ring); two consumer
//   warpgroups own 64 rows of X each:
//     S   = X . Y^T          wgmma SS-mode, hi/lo fp16 split operands (3 MMAs per K16), fp32 in registers
//     G   = (exp(S/T - lse_q) - diag) * w_q     computed on the register fragment and split into fp16 hi/lo, which is
//                                               exactly the register layout of a wgmma A operand
//     dX += G . Y            wgmma RS-mode: G from registers, Y straight from the same smem tile as an MN-major operand
//   launch 1: X = q, Y = c  -> dq ;  launch 2: X = c, Y = q (lse/w become per-column vectors staged with the tile) -> dc.
// The [B,C] logits / probabilities never touch HBM; the scores are the same split products as the forward pass
// (softmax_tc.cu), so exp(s - lse) is consistent with the saved lse.  d <= 64.
#include <cuda_fp16.h>
#include "common.cuh"
#include "tc_ptx.cuh"
#include "tc_split.cuh"
#include "softmax_ext.cuh"

namespace tfrs {
namespace tc {

constexpr int SB_THREADS = 288;                // warpgroups 0-1: MMA + transform, warp 8: bulk-TMA producer
constexpr int SB_STAGES = 4;
// the tensor core's fp32 adder truncates: a chain of thousands of accumulations into the same accumulator drifts (5e-5
// of the gradient scale at C = 16384), so each chain restarts every SB_DRAIN streamed tiles = 192 accumulation steps
// (the length of the forward Cross chain) and is added into an fp32 register sum (round-to-nearest adds)
constexpr int SB_DRAIN = 8;
constexpr int SB_Y_BYTES = 32768;              // one 128-row tile: hi 16 KB | lo 16 KB
constexpr int SB_STAGE_BYTES = SB_Y_BYTES + 1024;  // + lse[128] | w[128] of the tile (transposed launch)
constexpr float SB_LOG2E = 1.4426950408889634f;

struct SoftmaxBwdParams {
  const unsigned char* ximg; const unsigned char* yimg;
  const CxStats* xst; const CxStats* yst; const CxStats* wst;
  const float* lse_pad; const float* w_pad;   // indexed by QUERY, padded to a multiple of 128 (w already * 2^wst.exp)
  const float* grad_loss;
  const float* cbias_pad;                     // BIAS: per-CANDIDATE logit bias (natural units), padded to a multiple of 128
  long long n_x_rows, n_y_valid, n_ytiles, part_stride;
  int n_xb, parts, d;
  float inv_t;
  float* out;
  // EXT (accidental-hit removal / score_mask, see softmax_tc.cu): masked entries get G = 0
  const int* id_lo; const int* id_hi;   // candidate ids (32-bit halves, padded); query j's positive is candidate j
  const uint32_t* mbits; int mwords;    // keep-bits [stationary row][streamed column]: the (B,C) matrix for dq, its transpose for dc
};

__device__ __forceinline__ uint32_t pack_half2(float a, float b) {
  const __half2 h = __floats2half2_rn(a, b);
  return *reinterpret_cast<const uint32_t*>(&h);
}

template <bool TRANSPOSED, int MODE>
__global__ void __launch_bounds__(SB_THREADS, 1)
softmax_tc_bwd_kernel(const SoftmaxBwdParams p) {
  constexpr bool BIAS = MODE >= 1;
  constexpr bool EXT = MODE == 2;
  extern __shared__ __align__(1024) unsigned char sb_raw[];
  unsigned char* smem = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(sb_raw) + 1023) & ~uintptr_t(1023));
  unsigned char* sX = smem;                       // 32 KB
  unsigned char* sY = smem + 32768;               // SB_STAGES x SB_STAGE_BYTES
  uint64_t* bars = reinterpret_cast<uint64_t*>(sY + SB_STAGES * SB_STAGE_BYTES);
  uint64_t* y_full = bars;
  uint64_t* y_empty = bars + SB_STAGES;
  uint64_t* x_full = bars + 2 * SB_STAGES;

  const int wg = threadIdx.x >> 7, warp = (threadIdx.x >> 5) & 3, lane = threadIdx.x & 31;
  const int xb = blockIdx.x % p.n_xb, part = blockIdx.x / p.n_xb;
  const long long t_begin = (long long)part * p.n_ytiles / p.parts;
  const long long t_end = (long long)(part + 1) * p.n_ytiles / p.parts;
  const int n_iter = (int)(t_end - t_begin);

  if (threadIdx.x == 0) {
    for (int s = 0; s < SB_STAGES; ++s) { mbar_init(&y_full[s], 1); mbar_init(&y_empty[s], 8); }
    mbar_init(x_full, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (wg == 2) {
    if (threadIdx.x == 256) {
      mbar_expect_tx(x_full, 32768);
      bulk_g2s(sX, p.ximg + (long long)xb * 32768, 32768, x_full);
      int stage = 0; uint32_t phase = 0;
      for (int it = 0; it < n_iter; ++it) {
        mbar_wait(&y_empty[stage], phase ^ 1);
        unsigned char* dst = sY + stage * SB_STAGE_BYTES;
        const long long tile = t_begin + it;
        mbar_expect_tx(&y_full[stage], TRANSPOSED ? SB_STAGE_BYTES : SB_Y_BYTES);
        bulk_g2s(dst, p.yimg + tile * SB_Y_BYTES, SB_Y_BYTES, &y_full[stage]);
        if (TRANSPOSED) {
          bulk_g2s(dst + SB_Y_BYTES, p.lse_pad + tile * 128, 512, &y_full[stage]);
          bulk_g2s(dst + SB_Y_BYTES + 512, p.w_pad + tile * 128, 512, &y_full[stage]);
        }
        if (++stage == SB_STAGES) { stage = 0; phase ^= 1; }
      }
    }
    return;
  }
  // warpgroup c: stationary rows [64 c, 64 c + 64) of the 128-row block; a thread holds rows r, r + 8 of the warp's 16
  const int c = wg;
  const long long row_a = (long long)xb * 128 + c * 64 + warp * 16 + (lane >> 2);
  const float scale = ldexpf(p.inv_t, -(p.xst->exp + p.yst->exp));  // accumulator -> logit (natural units)
  float lse_r[2] = {0.f, 0.f}, w_r[2] = {1.f, 1.f}, bias_r[2] = {0.f, 0.f};
  int rid_lo[2] = {0, 0}, rid_hi[2] = {0, 0};   // id of the stationary row: the positive's id of query `row` (dq) / candidate `row` (dc)
#pragma unroll
  for (int rr = 0; rr < 2; ++rr) {
    const long long row = row_a + 8 * rr;   // padded arrays: in range for every row of the block
    if (BIAS && TRANSPOSED) bias_r[rr] = p.cbias_pad[row];
    if (!TRANSPOSED) {
      lse_r[rr] = p.lse_pad[row] - 14.0f * 0.6931471805599453f;  // folds the 2^14 fp16 range scale into the exponent
      w_r[rr] = p.w_pad[row];                                     // w_i * 2^wst.exp, applied to the dX row at the end
    }
    if (EXT && p.id_lo) { rid_lo[rr] = p.id_lo[row]; rid_hi[rr] = p.id_hi[row]; }
  }
  float dacc[32];   // fp32 sum of the drained chunks (round-to-nearest adds between tensor-core chains)
#pragma unroll
  for (int i = 0; i < 32; ++i) dacc[i] = 0.f;
  float dx[32];

  mbar_wait(x_full, 0);
  const uint32_t xa = smem_u32(sX) + c * 8192;
  const uint64_t x_hi = make_smem_desc(xa), x_lo = make_smem_desc(xa + 16384);
  for (int it = 0; it < n_iter; ++it) {
    const int stage = it % SB_STAGES;
    mbar_wait(&y_full[stage], (uint32_t)((it / SB_STAGES) & 1));
    const uint32_t y0 = smem_u32(sY + stage * SB_STAGE_BYTES);
    const uint64_t y_hi = make_smem_desc(y0), y_lo = make_smem_desc(y0 + 16384);
    // S = X . Y^T: the same three products, in the same order, as the forward pass (q_hi c_hi, q_lo c_hi, q_hi c_lo)
    float acc[64];
    wgmma_fence();
#pragma unroll
    for (int k4 = 0; k4 < 4; ++k4) {
      const uint64_t o = (uint64_t)(k4 * 2);
      wgmma_m64n128_ss(acc, x_hi + o, y_hi + o, (uint32_t)(k4 != 0));
      if (TRANSPOSED) {
        wgmma_m64n128_ss(acc, x_hi + o, y_lo + o, 1u);
        wgmma_m64n128_ss(acc, x_lo + o, y_hi + o, 1u);
      } else {
        wgmma_m64n128_ss(acc, x_lo + o, y_hi + o, 1u);
        wgmma_m64n128_ss(acc, x_hi + o, y_lo + o, 1u);
      }
    }
    wgmma_commit();
    wgmma_wait<0>();
    acc_fence(acc);

    // G = (exp(s/T - lse) - diag) * weight, masked entries 0 (see the header); then hi/lo fp16 as wgmma A fragments
    const long long col0 = (t_begin + it) * 128;
    const float* lse_s = reinterpret_cast<const float*>(sY + stage * SB_STAGE_BYTES + SB_Y_BYTES);   // TRANSPOSED
    const float* w_s = lse_s + 128;
    uint32_t ghi[32], glo[32];
#pragma unroll
    for (int i = 0; i < 64; i += 2) {
      const int rr = (i >> 1) & 1;
      const long long row = row_a + 8 * rr;
      float a[2];
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int cl = frag_col(i + e, lane);
        const long long col = col0 + cl;
        float lq = lse_r[rr], wq = 16384.f;
        if (TRANSPOSED) { lq = lse_s[cl]; wq = w_s[cl]; if (BIAS) lq -= bias_r[rr]; }
        else if (BIAS) lq -= __ldg(p.cbias_pad + col);
        float pr = ex2_approx(fmaf(acc[i + e], scale, -lq) * SB_LOG2E);
        if (TRANSPOSED) {
          if (col == row) pr -= 1.0f;
          pr *= wq;
        } else {
          if (col == row) pr -= 16384.f;
        }
        bool keep = col < p.n_y_valid;
        if (EXT) {
          if (p.mbits) keep &= ((__ldg(p.mbits + row * p.mwords + (t_begin + it) * 4 + (cl >> 5)) >> (cl & 31)) & 1u) != 0u;
          if (p.id_lo && __ldg(p.id_lo + col) == rid_lo[rr] && __ldg(p.id_hi + col) == rid_hi[rr] && col != row) keep = false;
        }
        a[e] = keep ? pr : 0.f;
      }
      const __half2 h = __floats2half2_rn(a[0], a[1]);
      const float2 hf = __half22float2(h);
      ghi[i >> 1] = *reinterpret_cast<const uint32_t*>(&h);
      glo[i >> 1] = pack_half2(a[0] - hf.x, a[1] - hf.y);
    }
    // dX += G . Y: K = the tile's 128 rows in 8 steps of 16; the Y tile is the MN-major B operand (d contiguous)
    const bool first = (it % SB_DRAIN) == 0;
    wgmma_fence();
#pragma unroll
    for (int kc = 0; kc < 8; ++kc) {
      const uint32_t ah[4] = {ghi[4 * kc], ghi[4 * kc + 1], ghi[4 * kc + 2], ghi[4 * kc + 3]};
      const uint32_t al[4] = {glo[4 * kc], glo[4 * kc + 1], glo[4 * kc + 2], glo[4 * kc + 3]};
      const uint64_t b_hi = make_smem_desc(y0 + kc * 2048), b_lo = make_smem_desc(y0 + 16384 + kc * 2048);
      wgmma_m64n64_rs_bmn(dx, ah, b_hi, (uint32_t)(!first || kc != 0));
      wgmma_m64n64_rs_bmn(dx, al, b_hi, 1u);
      wgmma_m64n64_rs_bmn(dx, ah, b_lo, 1u);
    }
    wgmma_commit();
    wgmma_wait<0>();
    acc_fence(dx);
    __syncwarp();
    if (lane == 0) mbar_arrive(&y_empty[stage]);
    if ((it % SB_DRAIN) == SB_DRAIN - 1 || it == n_iter - 1) {
#pragma unroll
      for (int i = 0; i < 32; ++i) dacc[i] += dx[i];
    }
  }
  const float gl = p.grad_loss ? p.grad_loss[0] : 1.0f;
#pragma unroll
  for (int rr = 0; rr < 2; ++rr) {
    const long long row = row_a + 8 * rr;
    if (row >= p.n_x_rows) continue;
    // transposed: G carried w^ = w 2^wexp per column; otherwise G carried 2^14 and the row weight is applied here
    const float f = TRANSPOSED ? gl * p.inv_t : gl * p.inv_t * w_r[rr];
    const int fe = TRANSPOSED ? -(p.wst->exp + p.yst->exp) : -(p.wst->exp + 14 + p.yst->exp);
    const float fs = ldexpf(f, fe);
    // a tiny operand or grad_loss can push the factor out of the normal range (dq near 2^-110 needs 2^-138) while the
    // gradient itself is normal: then it is applied as two normal factors, f 2^(fe - e2) and 2^e2, so that only the
    // final product rounds there.  Where fs is normal the second factor is 1 and the bits are those of dacc * fs.
    const bool fs_normal = fabsf(fs) >= 1.17549435e-38f && fabsf(fs) <= 3.40282347e38f;
    const int e2 = fs_normal ? 0 : min(max(fe, -126), 127);
    const float f1 = fs_normal ? fs : ldexpf(f, fe - e2), f2 = ldexpf(1.0f, e2);
    float* dst = p.out + (long long)part * p.part_stride + row * p.d;
#pragma unroll
    for (int i = 0; i < 32; ++i) {
      if (((i >> 1) & 1) != rr) continue;
      const int col = frag_col(i, lane);
      if (col < p.d) dst[col] = dacc[i] * f1 * f2;
    }
  }
}

// max |w| (1 when w == NULL) -> the exact power-of-two scale that puts it in [2^13, 2^14)
__global__ void __launch_bounds__(1024) sb_wstats_kernel(const float* __restrict__ w, long long B, CxStats* __restrict__ st) {
  __shared__ float red[32];
  float a = w ? 0.f : 1.0f;
  if (w) for (long long i = threadIdx.x; i < B; i += 1024) a = fmaxf(a, fabsf(w[i]));
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) a = fmaxf(a, __shfl_xor_sync(0xffffffffu, a, o));
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = a;
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int i = 1; i < 32; ++i) a = fmaxf(a, red[i]);
    int x = 0;
    const bool ok = a > 0.f && a < INFINITY;
    if (ok) (void)frexpf(a, &x);
    st->amax_bits = __float_as_uint(a);
    st->exp = ok ? (CX_TARGET_EXP - x) : 0;
  }
}
__global__ void __launch_bounds__(256)
sb_prep_kernel(const float* __restrict__ lse, const float* __restrict__ w, long long B, long long Bpad,
               const CxStats* __restrict__ wst, float* __restrict__ lse_pad, float* __restrict__ w_pad) {
  const long long i = (long long)blockIdx.x * 256 + threadIdx.x;
  if (i >= Bpad) return;
  lse_pad[i] = i < B ? lse[i] : 0.f;
  w_pad[i] = i < B ? ldexpf(w ? w[i] : 1.0f, wst->exp) : 0.f;
}
struct SbPlan {
  long long q_tiles, c_tiles; int parts_q, parts_c;
  size_t o_qst, o_cst, o_wst, o_qimg, o_cimg, o_lse, o_w, o_bias, o_partial, o_idlo, o_idhi, o_mbits, o_mbits_t, total;
};
static bool sb_plan(long long B, long long C, int d, SbPlan& pl, bool has_ids, bool has_mask) {
  if (B <= 0 || C < B || d <= 0 || d > 64) return false;
  pl.q_tiles = ceil_div(B, 128); pl.c_tiles = ceil_div(C, 128);
  pl.parts_q = stream_parts(pl.q_tiles, pl.c_tiles);   // dq: X = q blocks, Y = c tiles
  pl.parts_c = stream_parts(pl.c_tiles, pl.q_tiles);   // dc: X = c blocks, Y = q tiles
  size_t o = 0;
  auto take = [&](size_t bytes) { size_t r = o; o += align_up(bytes, 1024); return r; };
  pl.o_qst = take(sizeof(CxStats)); pl.o_cst = take(sizeof(CxStats)); pl.o_wst = take(sizeof(CxStats));
  pl.o_qimg = take((size_t)pl.q_tiles * 32768);
  pl.o_cimg = take((size_t)pl.c_tiles * 32768);
  pl.o_lse = take((size_t)pl.q_tiles * 128 * 4);
  pl.o_w = take((size_t)pl.q_tiles * 128 * 4);
  pl.o_bias = take((size_t)pl.c_tiles * 128 * 4);
  size_t pq = pl.parts_q > 1 ? (size_t)pl.parts_q * B * d * 4 : 0, pc = pl.parts_c > 1 ? (size_t)pl.parts_c * C * d * 4 : 0;
  pl.o_partial = take(pq > pc ? pq : pc);
  pl.o_idlo = take(has_ids ? (size_t)pl.c_tiles * 128 * 4 : 0);
  pl.o_idhi = take(has_ids ? (size_t)pl.c_tiles * 128 * 4 : 0);
  pl.o_mbits = take(has_mask ? (size_t)pl.q_tiles * 128 * pl.c_tiles * 4 * 4 : 0);     // [q rows][c words]
  pl.o_mbits_t = take(has_mask ? (size_t)pl.c_tiles * 128 * pl.q_tiles * 4 * 4 : 0);   // [c rows][q words]
  pl.total = o;
  return true;
}

}  // namespace tc
}  // namespace tfrs
using namespace tfrs;
using namespace tfrs::tc;

// pad[i] = src[i] for i < n, 0 on the padding
__global__ void __launch_bounds__(256) sb_pad_kernel(const float* __restrict__ src, long long n, long long npad, float* __restrict__ pad) {
  const long long i = (long long)blockIdx.x * 256 + threadIdx.x;
  if (i < npad) pad[i] = i < n ? src[i] : 0.f;
}

extern "C" size_t tfrs_inbatch_softmax_tc_bwd_workspace_bytes(int64_t B, int64_t C, int d, int has_ids, int has_mask) {
  SbPlan pl;
  return sb_plan(B, C, d, pl, has_ids != 0, has_mask != 0) ? pl.total : 0;
}

extern "C" int tfrs_inbatch_softmax_tc_bwd(const float* q, const float* c, int64_t B, int64_t C, int d, float inv_temperature,
                                           const float* sample_weight, const float* candidate_bias, const int64_t* candidate_ids,
                                           const uint8_t* score_mask, const float* lse, const float* grad_loss, float* dq, float* dc,
                                           void* ws, size_t ws_bytes, void* stream) {
  TFRS_CHECK_ARG(q && c && lse && dq && dc, "inbatch_softmax_tc_bwd: NULL pointer");
  SbPlan pl;
  const bool ext = candidate_ids || score_mask;
  if (!sb_plan(B, C, d, pl, candidate_ids != nullptr, score_mask != nullptr)) { set_error("inbatch_softmax_tc_bwd: shape outside the tensor-core path (need B <= C, d <= 64)"); return TFRS_ERR_UNSUPPORTED; }
  if (!ws || ws_bytes < pl.total) { set_error("inbatch_softmax_tc_bwd: workspace too small"); return TFRS_ERR_WORKSPACE_TOO_SMALL; }
  TFRS_CHECK_ARG((reinterpret_cast<uintptr_t>(ws) & 15) == 0, "inbatch_softmax_tc_bwd: workspace must be 16-byte aligned");
  cudaStream_t st = (cudaStream_t)stream;
  unsigned char* w8 = (unsigned char*)ws;
  CxStats* qst = (CxStats*)(w8 + pl.o_qst); CxStats* cst = (CxStats*)(w8 + pl.o_cst); CxStats* wst = (CxStats*)(w8 + pl.o_wst);
  unsigned char* qimg = w8 + pl.o_qimg; unsigned char* cimg = w8 + pl.o_cimg;
  float* lse_pad = (float*)(w8 + pl.o_lse); float* w_pad = (float*)(w8 + pl.o_w); float* partial = (float*)(w8 + pl.o_partial);
  TFRS_CUDA(cudaMemsetAsync(w8, 0, 3072, st));
  int rc = split_image(q, d, false, nullptr, B, d, 1, pl.q_tiles, qst, qimg, st);
  if (rc) return rc;
  rc = split_image(c, d, false, nullptr, C, d, 1, pl.c_tiles, cst, cimg, st);
  if (rc) return rc;
  sb_wstats_kernel<<<1, 1024, 0, st>>>(sample_weight, B, wst);
  TFRS_LAUNCH_CHECK();
  sb_prep_kernel<<<(unsigned)ceil_div(pl.q_tiles * 128, 256), 256, 0, st>>>(lse, sample_weight, B, pl.q_tiles * 128, wst, lse_pad, w_pad);
  TFRS_LAUNCH_CHECK();
  const size_t smem = 32768 + (size_t)SB_STAGES * SB_STAGE_BYTES + 1024 + 256;  // X | Y ring | align slack | barriers
  TFRS_DYN_SMEM((softmax_tc_bwd_kernel<false, 0>), (int)smem);
  TFRS_DYN_SMEM((softmax_tc_bwd_kernel<true, 0>), (int)smem);
  TFRS_DYN_SMEM((softmax_tc_bwd_kernel<false, 1>), (int)smem);
  TFRS_DYN_SMEM((softmax_tc_bwd_kernel<true, 1>), (int)smem);
  TFRS_DYN_SMEM((softmax_tc_bwd_kernel<false, 2>), (int)smem);
  TFRS_DYN_SMEM((softmax_tc_bwd_kernel<true, 2>), (int)smem);
  SoftmaxBwdParams p{};
  p.xst = qst; p.yst = cst; p.wst = wst; p.lse_pad = lse_pad; p.w_pad = w_pad; p.grad_loss = grad_loss; p.d = d; p.inv_t = inv_temperature;
  const int mode = ext ? 2 : (candidate_bias ? 1 : 0);
  if (mode) {   // EXT without a bias runs on a zero bias vector
    float* cbp = (float*)(w8 + pl.o_bias);
    if (candidate_bias) sb_pad_kernel<<<(unsigned)ceil_div(pl.c_tiles * 128, 256), 256, 0, st>>>(candidate_bias, C, pl.c_tiles * 128, cbp);
    else TFRS_CUDA(cudaMemsetAsync(cbp, 0, (size_t)pl.c_tiles * 128 * 4, st));
    TFRS_LAUNCH_CHECK();
    p.cbias_pad = cbp;
  }
  uint32_t* mbits = nullptr; uint32_t* mbits_t = nullptr;
  if (candidate_ids) {
    int* lo = (int*)(w8 + pl.o_idlo); int* hi = (int*)(w8 + pl.o_idhi);
    sx_ids_split_kernel<<<(unsigned)ceil_div(pl.c_tiles * 128, 256), 256, 0, st>>>((const long long*)candidate_ids, C, pl.c_tiles * 128, lo, hi);
    TFRS_LAUNCH_CHECK();
    p.id_lo = lo; p.id_hi = hi;
  }
  if (score_mask) {
    mbits = (uint32_t*)(w8 + pl.o_mbits); mbits_t = (uint32_t*)(w8 + pl.o_mbits_t);
    const int wc = (int)(pl.c_tiles * 4), wq = (int)(pl.q_tiles * 4);
    sx_mask_pack_kernel<<<(unsigned)ceil_div(pl.q_tiles * 128 * wc, 256), 256, 0, st>>>(score_mask, B, C, pl.q_tiles * 128, wc, mbits);
    TFRS_LAUNCH_CHECK();
    sx_mask_pack_t_kernel<<<dim3((unsigned)ceil_div(pl.c_tiles * 128, 256), (unsigned)wq), 256, 0, st>>>(score_mask, B, C, pl.c_tiles * 128, wq, mbits_t);
    TFRS_LAUNCH_CHECK();
  }
  // ---- dq: X = q, Y = c
  p.ximg = qimg; p.yimg = cimg; p.n_x_rows = B; p.n_y_valid = C; p.n_ytiles = pl.c_tiles; p.n_xb = (int)pl.q_tiles; p.parts = pl.parts_q;
  p.part_stride = B * (long long)d; p.out = pl.parts_q > 1 ? partial : dq;
  p.mbits = mbits; p.mwords = (int)(pl.c_tiles * 4);
  {
    const unsigned g = (unsigned)(pl.q_tiles * pl.parts_q);
    if (mode == 2) softmax_tc_bwd_kernel<false, 2><<<g, SB_THREADS, smem, st>>>(p);
    else if (mode == 1) softmax_tc_bwd_kernel<false, 1><<<g, SB_THREADS, smem, st>>>(p);
    else softmax_tc_bwd_kernel<false, 0><<<g, SB_THREADS, smem, st>>>(p);
  }
  TFRS_LAUNCH_CHECK();
  if (pl.parts_q > 1) {
    rc = reduce_parts(partial, B, d, pl.parts_q, dq, d, st);
    if (rc) return rc;
  }
  // ---- dc: X = c, Y = q (only the B query rows exist; candidates beyond B are pure negatives)
  p.ximg = cimg; p.yimg = qimg; p.xst = cst; p.yst = qst; p.n_x_rows = C; p.n_y_valid = B; p.n_ytiles = pl.q_tiles; p.n_xb = (int)pl.c_tiles;
  p.parts = pl.parts_c; p.part_stride = C * (long long)d; p.out = pl.parts_c > 1 ? partial : dc;
  p.mbits = mbits_t; p.mwords = (int)(pl.q_tiles * 4);
  {
    const unsigned g = (unsigned)(pl.c_tiles * pl.parts_c);
    if (mode == 2) softmax_tc_bwd_kernel<true, 2><<<g, SB_THREADS, smem, st>>>(p);
    else if (mode == 1) softmax_tc_bwd_kernel<true, 1><<<g, SB_THREADS, smem, st>>>(p);
    else softmax_tc_bwd_kernel<true, 0><<<g, SB_THREADS, smem, st>>>(p);
  }
  TFRS_LAUNCH_CHECK();
  return pl.parts_c > 1 ? reduce_parts(partial, C, d, pl.parts_c, dc, d, st) : TFRS_OK;
}
