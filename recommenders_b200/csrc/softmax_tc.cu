// softmax_tc.cu -- K3 forward on the tensor cores: in-batch sampled-softmax loss of tfrs.tasks.Retrieval
//   tasks/retrieval.py:178-180 (scores = q . c^T), :185 (labels = eye), :187-188 (/temperature), :210 + :86-87
//   loss = sum_i w_i * (logsumexp_j (q_i . c_j / T)  -  q_i . c_i / T)
// as ONE wgmma GEMM whose epilogue keeps an online (max, sum-exp) per query row and picks the diagonal --
// the [B,C] logits and the eye() labels never exist.  fp32 parity: hi/lo fp16 split of both operands (tc_split.cuh),
// 3 MMAs per K step, fp32 accumulation in registers (~2^-21 relative on a score).
//
// CTA shape = the top-K scan's: 256 query rows (two 128-row A blocks, hi+lo, resident), candidate tiles of
// 128 rows streamed through a bulk-TMA ring by one producer warp, 4 consumer warpgroups (64 query rows each,
// wgmma m64n128k16, the epilogue on the register fragment).  Grid = query blocks x candidate parts; every (row, part, column-half) leaves a partial
// (max, sum-exp) pair that `smtc_combine_kernel` folds into lse_i and the weighted row loss; the scalar loss is
// reduced in fixed order in fp64 (deterministic).  The backward pass (softmax.cu) consumes the same `lse`.
#include <cuda_fp16.h>
#include "common.cuh"
#include "tc_ptx.cuh"
#include "tc_split.cuh"
#include "softmax_ext.cuh"

namespace tfrs {
namespace tc {

constexpr int SX_THREADS = 544;
// candidate-tile ring depth: 4 x 32 KB at d <= 64, 1 x 64 KB at d <= 128 (A = 128 KB there)
__host__ __device__ constexpr int sx_stages(int kb) { return kb == 1 ? 4 : 1; }
constexpr float SX_LOG2E = 1.4426950408889634f;

struct SoftmaxTcParams {
  const unsigned char* qimg;  // [2*nqb tiles][kb][hi|lo][16 KB]
  const unsigned char* cimg;  // [n_ctiles][kb][hi|lo][16 KB]
  const CxStats* qst; const CxStats* cst;
  long long B, C;
  int nqb, parts, kb;
  long long n_ctiles;
  float inv_t;
  float2* partial;            // [Bp, parts, 2] (max, sum-exp) in log2 units
  float* pos;                 // [Bp] positive logit (q_i.c_i/T + bias_i, after the masks) in log2 units
  const float* cbias2;        // MODE >= 1: per-candidate logit bias in log2 units, padded to n_ctiles*128 (zeros beyond C)
  // MODE 2 (the remaining Retrieval options, each nullable):
  const int* id_lo; const int* id_hi;   // candidate ids split into 32-bit halves, padded: remove_accidental_hits
  const uint32_t* mbits; int mwords;    // score_mask as bits [Bp][mwords = n_ctiles*4] (1 = keep)
};

// MIN_FLOAT (layers/loss.py:23: float32 min / 100) in log2 units: the value a masked logit takes
constexpr float SX_MIN2 = -3.4028235e36f * SX_LOG2E;

// MODE 0: plain; 1: + per-candidate bias (sampling-probability correction); 2: + accidental-hit removal (candidate ids,
// tasks/retrieval.py:194-200, layers/loss.py:114-147: logits + dup * MIN_FLOAT == MIN_FLOAT in fp32) and score_mask
// (retrieval.py:202-203: where(mask, s, MIN_FLOAT)) applied to the accumulators in registers.
// (m, l) pairs in log2 units: merge b into a (an empty pair is m = -inf, l = 0)
__device__ __forceinline__ void lse_merge(float& m, float& l, float mb, float lb) {
  const float M = fmaxf(m, mb);
  if (M == -INFINITY) return;
  l = l * ex2_approx(m - M) + lb * ex2_approx(mb - M);
  m = M;
}

template <int KB, int MODE>
__global__ void __launch_bounds__(SX_THREADS, 1)
softmax_tc_kernel(const SoftmaxTcParams p) {
  constexpr bool BIAS = MODE >= 1;
  constexpr bool EXT = MODE == 2;
  extern __shared__ __align__(1024) unsigned char sx_raw[];
  unsigned char* smem = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(sx_raw) + 1023) & ~uintptr_t(1023));
  constexpr int SX_STAGES = sx_stages(KB);
  constexpr int A_BYTES = 2 * KB * 32768;      // two A blocks, hi+lo per K slab
  constexpr int B_BYTES = KB * 32768;          // one candidate tile, hi+lo per K slab
  unsigned char* sA = smem;
  unsigned char* sB = smem + A_BYTES;
  uint64_t* bars = reinterpret_cast<uint64_t*>(sB + SX_STAGES * B_BYTES);
  uint64_t* full = bars;
  uint64_t* empty = bars + SX_STAGES;
  uint64_t* a_full = bars + 2 * SX_STAGES;

  const int wg = threadIdx.x >> 7, warp = (threadIdx.x >> 5) & 3, lane = threadIdx.x & 31;
  const int qb = blockIdx.x % p.nqb, part = blockIdx.x / p.nqb;
  const long long t_begin = (long long)part * p.n_ctiles / p.parts;
  const long long t_end = (long long)(part + 1) * p.n_ctiles / p.parts;
  const int n_iter = (int)(t_end - t_begin);

  if (threadIdx.x == 0) {
    for (int s = 0; s < SX_STAGES; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], 16); }
    mbar_init(a_full, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (wg == 4) {
    if (threadIdx.x == 512) {
      mbar_expect_tx(a_full, A_BYTES);
      bulk_g2s(sA, p.qimg + (long long)qb * A_BYTES, A_BYTES, a_full);
      int stage = 0; uint32_t phase = 0;
      for (int it = 0; it < n_iter; ++it) {
        mbar_wait(&empty[stage], phase ^ 1);
        mbar_expect_tx(&full[stage], B_BYTES);
        bulk_g2s(sB + stage * B_BYTES, p.cimg + (t_begin + it) * (long long)B_BYTES, B_BYTES, &full[stage]);
        if (++stage == SX_STAGES) { stage = 0; phase ^= 1; }
      }
    }
    return;
  }
  // warpgroup c: query rows [64 c, 64 c + 64) of the CTA's 256 (half c & 1 of A block c / 2); a thread holds rows r, r + 8
  // x 32 columns of every tile and keeps an online (max, sum-exp) per (row, column half), merged over the quad at the end
  const int c = wg;
  const long long row_a = (long long)qb * 256 + c * 64 + warp * 16 + (lane >> 2);
  // logits in log2 units: s2 = acc * 2^-(eq+ec) * invT * log2(e)
  const float scale2 = ldexpf(p.inv_t * SX_LOG2E, -(p.qst->exp + p.cst->exp));
  float m2[4] = {-INFINITY, -INFINITY, -INFINITY, -INFINITY}, l[4] = {0.f, 0.f, 0.f, 0.f};   // s = 2 rr + half
  float pos2[2] = {0.f, 0.f};
  bool has_pos[2] = {false, false};
  int rid_lo[2] = {0, 0}, rid_hi[2] = {0, 0};   // id of each row's positive candidate (candidate `row`); arrays padded past Bp
  if (EXT && p.id_lo) {
#pragma unroll
    for (int rr = 0; rr < 2; ++rr) { rid_lo[rr] = p.id_lo[row_a + 8 * rr]; rid_hi[rr] = p.id_hi[row_a + 8 * rr]; }
  }
  mbar_wait(a_full, 0);
  const uint32_t a0 = smem_u32(sA + (c >> 1) * KB * 32768 + (c & 1) * 8192);
  int stage = 0; uint32_t phase = 0;
  for (int it = 0; it < n_iter; ++it) {
    const long long col0 = (t_begin + it) * 128;
    mbar_wait(&full[stage], phase);
    float acc[64];
    wgmma_fence();
#pragma unroll
    for (int kb = 0; kb < KB; ++kb) {
      const uint32_t b0 = smem_u32(sB + stage * B_BYTES + kb * 32768);
      const uint64_t a_hi = make_smem_desc(a0 + kb * 32768), a_lo = make_smem_desc(a0 + kb * 32768 + 16384);
      const uint64_t b_hi = make_smem_desc(b0), b_lo = make_smem_desc(b0 + 16384);
#pragma unroll
      for (int k4 = 0; k4 < 4; ++k4) {
        const uint64_t o = (uint64_t)(k4 * 2);
        wgmma_m64n128_ss(acc, a_hi + o, b_hi + o, (uint32_t)((kb | k4) != 0));
        wgmma_m64n128_ss(acc, a_lo + o, b_hi + o, 1u);
        wgmma_m64n128_ss(acc, a_hi + o, b_lo + o, 1u);
      }
    }
    wgmma_commit();
    wgmma_wait<0>();
    acc_fence(acc);
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty[stage]);
    if (++stage == SX_STAGES) { stage = 0; phase ^= 1; }

    // BIAS (sampling-probability correction, retrieval.py:190-192): logits s/T + b_j -> turned into log2-unit logits in
    // place (one FFMA with the per-candidate bias), the rest runs with scale 1.  EXT masks set MIN_FLOAT.
    if (BIAS || EXT) {
#pragma unroll
      for (int i = 0; i < 64; ++i) {
        const long long col = col0 + frag_col(i, lane);
        const int rr = (i >> 1) & 1;
        float v = acc[i];
        if (BIAS) v = fmaf(v, scale2, __ldg(p.cbias2 + col));
        if (EXT) {
          const long long row = row_a + 8 * rr;
          if (p.id_lo && __ldg(p.id_lo + col) == rid_lo[rr] && __ldg(p.id_hi + col) == rid_hi[rr] && col != row) v = SX_MIN2;
          if (p.mbits) {
            const int cl = frag_col(i, lane);
            const uint32_t mw = __ldg(p.mbits + row * p.mwords + (t_begin + it) * 4 + (cl >> 5));
            if (!((mw >> (cl & 31)) & 1u)) v = SX_MIN2;
          }
        }
        acc[i] = v;
      }
    }
    const float sc = BIAS ? 1.0f : scale2;
    const int n_valid = (int)min(128ll, p.C - col0);  // columns beyond C are zero-padded rows of the image
#pragma unroll
    for (int rr = 0; rr < 2; ++rr) {
      const long long row = row_a + 8 * rr;
      if (row >= col0 && row < col0 + 128) {   // the positive of query i is candidate i (retrieval.py:185)
#pragma unroll
        for (int i = 0; i < 64; ++i)
          if (((i >> 1) & 1) == rr && col0 + frag_col(i, lane) == row) { pos2[rr] = acc[i] * sc; has_pos[rr] = true; }
      }
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        float tmax = -INFINITY;
#pragma unroll
        for (int jj = 0; jj < 8; ++jj) {
          const int i = 4 * (8 * h + jj) + 2 * rr;
          if (frag_col(i, lane) < n_valid) tmax = fmaxf(tmax, acc[i]);
          if (frag_col(i + 1, lane) < n_valid) tmax = fmaxf(tmax, acc[i + 1]);
        }
        if (tmax == -INFINITY) continue;
        const int s = 2 * rr + h;
        const float m_new = fmaxf(m2[s], tmax * sc);
        float a0s = 0.f, a1s = 0.f;
#pragma unroll
        for (int jj = 0; jj < 8; ++jj) {
          const int i = 4 * (8 * h + jj) + 2 * rr;
          if (frag_col(i, lane) < n_valid) a0s += ex2_approx(fmaf(acc[i], sc, -m_new));
          if (frag_col(i + 1, lane) < n_valid) a1s += ex2_approx(fmaf(acc[i + 1], sc, -m_new));
        }
        l[s] = l[s] * ex2_approx(m2[s] - m_new) + (a0s + a1s);
        m2[s] = m_new;
      }
    }
  }
  // merge the quad's partial (max, sum-exp) pairs; the quad leader writes them
#pragma unroll
  for (int s = 0; s < 4; ++s) {
#pragma unroll
    for (int o = 1; o <= 2; o <<= 1) {
      const float mo = __shfl_xor_sync(0xffffffffu, m2[s], o), lo_ = __shfl_xor_sync(0xffffffffu, l[s], o);
      lse_merge(m2[s], l[s], mo, lo_);
    }
  }
#pragma unroll
  for (int rr = 0; rr < 2; ++rr) {
    const long long row = row_a + 8 * rr;
    if (row < p.B) {
      if ((lane & 3) == 0) {
        p.partial[(row * p.parts + part) * 2 + 0] = make_float2(m2[2 * rr], l[2 * rr]);
        p.partial[(row * p.parts + part) * 2 + 1] = make_float2(m2[2 * rr + 1], l[2 * rr + 1]);
      }
      if (has_pos[rr]) p.pos[row] = pos2[rr];   // exactly one thread of one part saw the diagonal column
    }
  }
}

// lse_i = ln2 * (M + log2(sum_p l_p 2^(m_p - M)));  rowloss_i = w_i (lse_i - pos_i), formed as ln2 * ((M - pos2_i) + log2 L)
// so that a row whose logits are ALL MIN_FLOAT (fully masked) still yields log(C), as the max-subtracted reference does
__global__ void __launch_bounds__(256)
smtc_combine_kernel(const float2* __restrict__ partial, int n_partials, const float* __restrict__ pos,
                    const float* __restrict__ w, long long B, float* __restrict__ lse, float* __restrict__ rowloss) {
  const long long row = (long long)blockIdx.x * 256 + threadIdx.x;
  if (row >= B) return;
  const float2* pp = partial + row * n_partials;
  float M = -INFINITY;
  for (int i = 0; i < n_partials; ++i) M = fmaxf(M, pp[i].x);
  float L = 0.f;
  for (int i = 0; i < n_partials; ++i) L += pp[i].y * exp2f(pp[i].x - M);
  const float lg = log2f(L);
  lse[row] = (M + lg) * 0.6931471805599453f;
  rowloss[row] = (w ? w[row] : 1.0f) * (((M - pos[row]) + lg) * 0.6931471805599453f);
}

struct SxPlan { int kb, nqb, parts; long long Bp, n_ctiles, idpad; size_t smem, o_qst, o_cst, o_qimg, o_cimg, o_partial, o_pos, o_rowloss, o_bias, o_idlo, o_idhi, o_mbits, total; };

static bool sx_plan(long long B, long long C, int d, SxPlan& pl, bool has_ids, bool has_mask) {
  if (B <= 0 || C < B || d <= 0 || d > 128) return false;
  pl.kb = (int)ceil_div(d, 64);
  pl.nqb = (int)ceil_div(B, 256);
  pl.Bp = (long long)pl.nqb * 256;
  pl.n_ctiles = ceil_div(C, 128);
  pl.parts = stream_parts(pl.nqb, pl.n_ctiles);
  pl.smem = (size_t)(2 + sx_stages(pl.kb)) * pl.kb * 32768 + 1024 + 256;
  if (pl.smem > 227 * 1024) return false;
  size_t o = 0;
  auto take = [&](size_t bytes) { size_t r = o; o += align_up(bytes, 1024); return r; };
  pl.o_qst = take(sizeof(CxStats)); pl.o_cst = take(sizeof(CxStats));
  pl.o_qimg = take(cx_img_bytes(pl.Bp, d));
  pl.o_cimg = take(cx_img_bytes(pl.n_ctiles * 128, d));
  pl.o_partial = take((size_t)pl.Bp * pl.parts * 2 * sizeof(float2));
  pl.o_pos = take((size_t)pl.Bp * 4);
  pl.o_rowloss = take((size_t)pl.Bp * 4);
  pl.o_bias = take((size_t)pl.n_ctiles * 128 * 4);
  pl.idpad = pl.Bp > pl.n_ctiles * 128 ? pl.Bp : pl.n_ctiles * 128;
  pl.o_idlo = take(has_ids ? (size_t)pl.idpad * 4 : 0);
  pl.o_idhi = take(has_ids ? (size_t)pl.idpad * 4 : 0);
  pl.o_mbits = take(has_mask ? (size_t)pl.Bp * pl.n_ctiles * 4 * 4 : 0);
  pl.total = o;
  return true;
}

}  // namespace tc
}  // namespace tfrs
using namespace tfrs;
using namespace tfrs::tc;

// cbias2[i] = bias[i] * log2(e) for i < C, 0 on the padding (and everywhere when bias == NULL)
__global__ void __launch_bounds__(256)
smtc_bias_kernel(const float* __restrict__ bias, long long C, long long Cpad, float* __restrict__ cbias2) {
  const long long i = (long long)blockIdx.x * 256 + threadIdx.x;
  if (i < Cpad) cbias2[i] = (bias && i < C) ? bias[i] * SX_LOG2E : 0.f;
}

extern "C" size_t tfrs_inbatch_softmax_tc_workspace_bytes(int64_t B, int64_t C, int d, int has_ids, int has_mask) {
  SxPlan pl;
  return sx_plan(B, C, d, pl, has_ids != 0, has_mask != 0) ? pl.total : 0;
}

extern "C" int tfrs_inbatch_softmax_tc_fwd(const float* q, const float* c, int64_t B, int64_t C, int d, float inv_temperature,
                                           const float* sample_weight, const float* candidate_bias, const int64_t* candidate_ids,
                                           const uint8_t* score_mask, float* loss, float* lse, void* ws, size_t ws_bytes,
                                           void* stream) {
  TFRS_CHECK_ARG(q && c && loss && lse, "inbatch_softmax_tc_fwd: NULL pointer");
  SxPlan pl;
  const bool ext = candidate_ids || score_mask;
  if (!(inv_temperature > 0.f)) { set_error("inbatch_softmax_tc_fwd: needs a positive temperature"); return TFRS_ERR_UNSUPPORTED; }
  if (!sx_plan(B, C, d, pl, candidate_ids != nullptr, score_mask != nullptr)) { set_error("inbatch_softmax_tc_fwd: shape outside the tensor-core path (need B <= C, d <= 128)"); return TFRS_ERR_UNSUPPORTED; }
  if (!ws || ws_bytes < pl.total) { set_error("inbatch_softmax_tc_fwd: workspace too small"); return TFRS_ERR_WORKSPACE_TOO_SMALL; }
  TFRS_CHECK_ARG((reinterpret_cast<uintptr_t>(ws) & 15) == 0, "inbatch_softmax_tc_fwd: workspace must be 16-byte aligned");
  cudaStream_t st = (cudaStream_t)stream;
  unsigned char* w = (unsigned char*)ws;
  CxStats* qst = (CxStats*)(w + pl.o_qst); CxStats* cst = (CxStats*)(w + pl.o_cst);
  unsigned char* qimg = w + pl.o_qimg; unsigned char* cimg = w + pl.o_cimg;
  float2* partial = (float2*)(w + pl.o_partial);
  float* pos = (float*)(w + pl.o_pos); float* rowloss = (float*)(w + pl.o_rowloss);
  TFRS_CUDA(cudaMemsetAsync(w, 0, 2048, st));  // both stats blocks
  int rc = split_image(q, d, false, nullptr, B, d, pl.kb, pl.Bp / 128, qst, qimg, st);
  if (rc) return rc;
  rc = split_image(c, d, false, nullptr, C, d, pl.kb, pl.n_ctiles, cst, cimg, st);
  if (rc) return rc;
  SoftmaxTcParams p{};
  p.qimg = qimg; p.cimg = cimg; p.qst = qst; p.cst = cst; p.B = B; p.C = C; p.nqb = pl.nqb; p.parts = pl.parts; p.kb = pl.kb;
  p.n_ctiles = pl.n_ctiles; p.inv_t = inv_temperature; p.partial = partial; p.pos = pos;
  const int s1 = (int)((2 + sx_stages(1)) * 32768 + 1280), s2 = (int)((2 + sx_stages(2)) * 2 * 32768 + 1280);
  TFRS_DYN_SMEM((softmax_tc_kernel<1, 0>), s1);
  TFRS_DYN_SMEM((softmax_tc_kernel<2, 0>), s2);
  TFRS_DYN_SMEM((softmax_tc_kernel<1, 1>), s1);
  TFRS_DYN_SMEM((softmax_tc_kernel<2, 1>), s2);
  TFRS_DYN_SMEM((softmax_tc_kernel<1, 2>), s1);
  TFRS_DYN_SMEM((softmax_tc_kernel<2, 2>), s2);
  const unsigned grid = (unsigned)(pl.nqb * pl.parts);
  if (candidate_bias || ext) {
    float* cb2 = (float*)(w + pl.o_bias);
    smtc_bias_kernel<<<(unsigned)ceil_div(pl.n_ctiles * 128, 256), 256, 0, st>>>(candidate_bias, C, pl.n_ctiles * 128, cb2);
    TFRS_LAUNCH_CHECK();
    p.cbias2 = cb2;
  }
  if (candidate_ids) {
    int* lo = (int*)(w + pl.o_idlo); int* hi = (int*)(w + pl.o_idhi);
    sx_ids_split_kernel<<<(unsigned)ceil_div(pl.idpad, 256), 256, 0, st>>>((const long long*)candidate_ids, C, pl.idpad, lo, hi);
    TFRS_LAUNCH_CHECK();
    p.id_lo = lo; p.id_hi = hi;
  }
  if (score_mask) {
    uint32_t* mb = (uint32_t*)(w + pl.o_mbits);
    p.mwords = (int)(pl.n_ctiles * 4);
    sx_mask_pack_kernel<<<(unsigned)ceil_div(pl.Bp * p.mwords, 256), 256, 0, st>>>(score_mask, B, C, pl.Bp, p.mwords, mb);
    TFRS_LAUNCH_CHECK();
    p.mbits = mb;
  }
  if (ext) {
    if (pl.kb == 1) softmax_tc_kernel<1, 2><<<grid, SX_THREADS, pl.smem, st>>>(p);
    else softmax_tc_kernel<2, 2><<<grid, SX_THREADS, pl.smem, st>>>(p);
  } else if (candidate_bias) {
    if (pl.kb == 1) softmax_tc_kernel<1, 1><<<grid, SX_THREADS, pl.smem, st>>>(p);
    else softmax_tc_kernel<2, 1><<<grid, SX_THREADS, pl.smem, st>>>(p);
  } else {
    if (pl.kb == 1) softmax_tc_kernel<1, 0><<<grid, SX_THREADS, pl.smem, st>>>(p);
    else softmax_tc_kernel<2, 0><<<grid, SX_THREADS, pl.smem, st>>>(p);
  }
  TFRS_LAUNCH_CHECK();
  smtc_combine_kernel<<<(unsigned)ceil_div(B, 256), 256, 0, st>>>(partial, pl.parts * 2, pos, sample_weight, B, lse, rowloss);
  TFRS_LAUNCH_CHECK();
  return reduce_loss(rowloss, B, 1, loss, st);
}
