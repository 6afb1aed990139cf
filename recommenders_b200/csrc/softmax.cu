// softmax.cu -- K3/K3b: in-batch sampled-softmax loss of tfrs.tasks.Retrieval and its backward.
//   tasks/retrieval.py:178-180 (scores = q . c^T), :185 (labels = eye), :187-188 (/temperature),
//   :210 + :86-87 (CategoricalCrossentropy(from_logits=True, reduction=SUM), sample_weight).
// The [B,C] logits are never materialised as a whole: rows are processed in blocks that stay
// L2-resident (<= 128 MB), labels are never built (the positive of row i is column i).
//   fwd: S_blk = exact SGEMM -> per-row max / sum-exp -> lse_i, row loss w_i*(lse_i - s_ii)
//        -> fixed-order fp64 reduction to the scalar loss (deterministic).
//   bwd: S_blk recomputed -> G = (exp(s - lse) - [j==i]) * w_i * grad_loss * invT (in place)
//        -> dq_blk = G . c ;  dc (+)= G^T . q_blk   (exact SGEMMs, one owner thread per output).
#include "sgemm.cuh"

namespace tfrs {

constexpr int SM_THREADS = 256;

__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// one CTA per row of the block
__global__ void __launch_bounds__(SM_THREADS)
sm_row_lse(const float* __restrict__ S, long long ldS, int C, long long row0, float invT,
           const float* __restrict__ w, float* __restrict__ lse, float* __restrict__ rowloss) {
  __shared__ float red[SM_THREADS / 32];
  __shared__ float bcast;
  const int r = blockIdx.x;
  const float* s = S + (long long)r * ldS;
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  float m = -INFINITY;
  for (int j = tid; j < C; j += SM_THREADS) m = fmaxf(m, s[j] * invT);
  m = warp_max(m);
  if (lane == 0) red[wid] = m;
  __syncthreads();
  if (tid == 0) { float v = red[0]; for (int i = 1; i < SM_THREADS / 32; ++i) v = fmaxf(v, red[i]); bcast = v; }
  __syncthreads();
  m = bcast;
  float sum = 0.f;
  for (int j = tid; j < C; j += SM_THREADS) sum += expf(s[j] * invT - m);
  sum = warp_sum(sum);
  __syncthreads();
  if (lane == 0) red[wid] = sum;
  __syncthreads();
  if (tid == 0) {
    float v = 0.f; for (int i = 0; i < SM_THREADS / 32; ++i) v += red[i];
    float l = m + logf(v);
    long long gi = row0 + r;
    lse[gi] = l;
    float pos = s[gi] * invT;  // the positive of query i is candidate i (retrieval.py:185)
    float wi = w ? w[gi] : 1.0f;
    rowloss[gi] = wi * (l - pos);
  }
}

// one CTA per row of the block: G = (exp(s - lse) - [j == i]) * w_i * grad_loss * invT, in place
__global__ void __launch_bounds__(SM_THREADS)
sm_make_grad(float* __restrict__ S, long long ldS, int C, int R, long long row0, float invT,
             const float* __restrict__ w, const float* __restrict__ lse, const float* __restrict__ grad_loss) {
  const int r = blockIdx.x;
  if (r >= R) return;
  const long long gi = row0 + r;
  const float gl = grad_loss ? grad_loss[0] : 1.0f;
  const float scale = (w ? w[gi] : 1.0f) * gl * invT;
  const float l = lse[gi];
  float* s = S + (long long)r * ldS;
  for (int j = threadIdx.x; j < C; j += SM_THREADS) {
    float p = expf(s[j] * invT - l);
    if (j == gi) p -= 1.0f;
    s[j] = p * scale;
  }
}

// ---- multi-head queries (tasks/retrieval.py:172-176): scores_ij = max_h q_ih . c_j ("maxsim").  The block's S holds the H
// head rows of a query consecutively (q is [B,H,d] flattened); one CTA per query folds them on the fly.
__global__ void __launch_bounds__(SM_THREADS)
sm_row_lse_maxsim(const float* __restrict__ S, long long ldS, int C, int H, long long q0, float invT,
                  const float* __restrict__ w, float* __restrict__ lse, float* __restrict__ rowloss) {
  __shared__ float red[SM_THREADS / 32];
  __shared__ float bcast;
  const int r = blockIdx.x;
  const float* s = S + (long long)r * H * ldS;
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  auto msim = [&](int j) { float v = s[j]; for (int h = 1; h < H; ++h) v = fmaxf(v, s[(long long)h * ldS + j]); return v * invT; };
  float m = -INFINITY;
  for (int j = tid; j < C; j += SM_THREADS) m = fmaxf(m, msim(j));
  m = warp_max(m);
  if (lane == 0) red[wid] = m;
  __syncthreads();
  if (tid == 0) { float v = red[0]; for (int i = 1; i < SM_THREADS / 32; ++i) v = fmaxf(v, red[i]); bcast = v; }
  __syncthreads();
  m = bcast;
  float sum = 0.f;
  for (int j = tid; j < C; j += SM_THREADS) sum += expf(msim(j) - m);
  sum = warp_sum(sum);
  __syncthreads();
  if (lane == 0) red[wid] = sum;
  __syncthreads();
  if (tid == 0) {
    float v = 0.f; for (int i = 0; i < SM_THREADS / 32; ++i) v += red[i];
    const float l = m + logf(v);
    const long long gi = q0 + r;
    lse[gi] = l;
    rowloss[gi] = (w ? w[gi] : 1.0f) * (l - msim((int)gi));   // the positive of query i is candidate i (retrieval.py:185)
  }
}

// G_ij = (exp(maxsim_ij/T - lse_i) - [j == i]) * w_i * grad_loss / T goes to the head(s) that attain the maximum -- split
// evenly among exact ties, as tf.reduce_max's gradient does -- and 0 to the others; written in place over the H score rows.
__global__ void __launch_bounds__(SM_THREADS)
sm_make_grad_maxsim(float* __restrict__ S, long long ldS, int C, int H, long long q0, float invT,
                    const float* __restrict__ w, const float* __restrict__ lse, const float* __restrict__ grad_loss) {
  const int r = blockIdx.x;
  const long long gi = q0 + r;
  const float gl = grad_loss ? grad_loss[0] : 1.0f;
  const float scale = (w ? w[gi] : 1.0f) * gl * invT;
  const float l = lse[gi];
  float* s = S + (long long)r * H * ldS;
  for (int j = threadIdx.x; j < C; j += SM_THREADS) {
    float mx = s[j];
    for (int h = 1; h < H; ++h) mx = fmaxf(mx, s[(long long)h * ldS + j]);
    int cnt = 0;
    for (int h = 0; h < H; ++h) cnt += (s[(long long)h * ldS + j] == mx) ? 1 : 0;
    float p = expf(mx * invT - l);
    if (j == gi) p -= 1.0f;
    const float g = p * scale / (float)cnt;
    for (int h = 0; h < H; ++h) {
      float* e = s + (long long)h * ldS + j;
      *e = (*e == mx) ? g : 0.f;
    }
  }
}

struct EpiAccum {  // C[m*ldc+n] (+)= v
  float* C; long long ldc; bool accumulate;
  __device__ __forceinline__ void operator()(int m, int n, float v, int) const {
    float* p = C + (long long)m * ldc + n;
    *p = accumulate ? (*p + v) : v;
  }
};

static long long sm_rows_per_block(long long B, long long C) {
  long long r = ((long long)128 << 20) / (C * 4);
  r = r / 128 * 128;
  if (r < 128) r = 128;
  if (r > B) r = B;
  return r;
}

}  // namespace tfrs
using namespace tfrs;

constexpr int SM_DQ_SPLITS = 8;  // dq = G . c is skinny (N = d): split K = C so that all SMs have work

extern "C" size_t tfrs_inbatch_softmax_workspace_bytes(int64_t B, int64_t C, int d) {
  if (B <= 0 || C <= 0) return 256;
  long long R = sm_rows_per_block(B, C);
  return align_up((size_t)R * C * 4, 256) + align_up((size_t)B * 4, 256) + align_up((size_t)SM_DQ_SPLITS * R * d * 4, 256);
}

static int sm_check(const float* q, const float* c, int64_t B, int64_t C, int d, void* ws, size_t ws_bytes) {
  TFRS_CHECK_ARG(q && c && B > 0 && C >= B && d > 0, "inbatch_softmax: need q, c, 0 < B <= C, d > 0");
  TFRS_CHECK_ARG(C < (1ll << 31) && B < (1ll << 31), "inbatch_softmax: B/C too large");
  if (!ws || ws_bytes < tfrs_inbatch_softmax_workspace_bytes(B, C, d)) {
    set_error("inbatch_softmax: workspace too small");
    return TFRS_ERR_WORKSPACE_TOO_SMALL;
  }
  return TFRS_OK;
}

extern "C" int tfrs_inbatch_softmax_fwd(const float* q, const float* c, int64_t B, int64_t C, int d,
                                        float inv_temperature, const float* sample_weight, float* loss,
                                        float* lse, void* ws, size_t ws_bytes, void* stream) {
  int rc = sm_check(q, c, B, C, d, ws, ws_bytes);
  if (rc) return rc;
  TFRS_CHECK_ARG(loss && lse, "inbatch_softmax_fwd: NULL output");
  cudaStream_t st = (cudaStream_t)stream;
  const long long R = sm_rows_per_block(B, C);
  float* S = (float*)ws;
  float* rowloss = (float*)((unsigned char*)ws + align_up((size_t)R * C * 4, 256));
  for (long long r0 = 0; r0 < B; r0 += R) {
    int rows = (int)((B - r0) < R ? (B - r0) : R);
    rc = launch_sgemm<false, true>(q + r0 * d, d, c, d, rows, (int)C, d, 1, EpiStore{S, C}, st);
    if (rc) return rc;
    sm_row_lse<<<rows, SM_THREADS, 0, st>>>(S, C, (int)C, r0, inv_temperature, sample_weight, lse, rowloss);
    TFRS_LAUNCH_CHECK();
  }
  return reduce_loss(rowloss, B, 1, loss, st);
}

extern "C" int tfrs_inbatch_softmax_bwd(const float* q, const float* c, int64_t B, int64_t C, int d,
                                        float inv_temperature, const float* sample_weight, const float* lse,
                                        const float* grad_loss, float* dq, float* dc, void* ws, size_t ws_bytes,
                                        void* stream) {
  int rc = sm_check(q, c, B, C, d, ws, ws_bytes);
  if (rc) return rc;
  TFRS_CHECK_ARG(lse && dq && dc, "inbatch_softmax_bwd: NULL pointer");
  cudaStream_t st = (cudaStream_t)stream;
  const long long R = sm_rows_per_block(B, C);
  float* S = (float*)ws;
  for (long long r0 = 0; r0 < B; r0 += R) {
    int rows = (int)((B - r0) < R ? (B - r0) : R);
    rc = launch_sgemm<false, true>(q + r0 * d, d, c, d, rows, (int)C, d, 1, EpiStore{S, C}, st);
    if (rc) return rc;
    sm_make_grad<<<(unsigned)rows, SM_THREADS, 0, st>>>(S, C, (int)C, rows, r0, inv_temperature, sample_weight, lse, grad_loss);
    TFRS_LAUNCH_CHECK();
    // dq[r0:r0+rows] = G . c      (M=rows, N=d, K=C; A=G row-major, B=c [C,d] not transposed); deterministic split-K
    float* part = (float*)((unsigned char*)ws + align_up((size_t)R * C * 4, 256) + align_up((size_t)B * 4, 256));
    rc = launch_sgemm_split_k<false, false>(S, C, c, d, rows, d, (int)C, SM_DQ_SPLITS, part, dq + r0 * d, st);
    if (rc) return rc;
    // dc (+)= G^T . q_blk         (M=C, N=d, K=rows; A=G read transposed)
    rc = launch_sgemm<true, false>(S, C, q + r0 * d, d, (int)C, d, rows, 1, EpiAccum{dc, d, r0 > 0}, st);
    if (rc) return rc;
  }
  return TFRS_OK;
}

// ---- multi-head (maxsim) variant: q is [B,H,d]; same row-block scheme on the B*H flattened query rows ----------------------
static long long smx_queries_per_block(long long B, int H, long long C) {
  long long r = sm_rows_per_block(B * H, C) / H;
  if (r < 1) r = 1;
  return r > B ? B : r;
}

extern "C" size_t tfrs_inbatch_softmax_maxsim_workspace_bytes(int64_t B, int H, int64_t C, int d) {
  if (B <= 0 || C <= 0 || H <= 0) return 256;
  const long long R = smx_queries_per_block(B, H, C) * H;
  return align_up((size_t)R * C * 4, 256) + align_up((size_t)B * 4, 256) + align_up((size_t)SM_DQ_SPLITS * R * d * 4, 256);
}

extern "C" int tfrs_inbatch_softmax_maxsim_fwd(const float* q, const float* c, int64_t B, int H, int64_t C, int d,
                                               float inv_temperature, const float* sample_weight, float* loss, float* lse,
                                               void* ws, size_t ws_bytes, void* stream) {
  TFRS_CHECK_ARG(q && c && loss && lse && B > 0 && H > 0 && C >= B && d > 0, "inbatch_softmax_maxsim_fwd: bad arguments");
  TFRS_CHECK_ARG(C < (1ll << 31) && B * H < (1ll << 31), "inbatch_softmax_maxsim_fwd: B*H / C too large");
  if (!ws || ws_bytes < tfrs_inbatch_softmax_maxsim_workspace_bytes(B, H, C, d)) { set_error("inbatch_softmax_maxsim: workspace too small"); return TFRS_ERR_WORKSPACE_TOO_SMALL; }
  cudaStream_t st = (cudaStream_t)stream;
  const long long Rq = smx_queries_per_block(B, H, C);
  float* S = (float*)ws;
  float* rowloss = (float*)((unsigned char*)ws + align_up((size_t)Rq * H * C * 4, 256));
  for (long long q0 = 0; q0 < B; q0 += Rq) {
    const int nq = (int)((B - q0) < Rq ? (B - q0) : Rq);
    int rc = launch_sgemm<false, true>(q + q0 * H * d, d, c, d, nq * H, (int)C, d, 1, EpiStore{S, C}, st);
    if (rc) return rc;
    sm_row_lse_maxsim<<<nq, SM_THREADS, 0, st>>>(S, C, (int)C, H, q0, inv_temperature, sample_weight, lse, rowloss);
    TFRS_LAUNCH_CHECK();
  }
  return reduce_loss(rowloss, B, 1, loss, st);
}

extern "C" int tfrs_inbatch_softmax_maxsim_bwd(const float* q, const float* c, int64_t B, int H, int64_t C, int d,
                                               float inv_temperature, const float* sample_weight, const float* lse,
                                               const float* grad_loss, float* dq, float* dc, void* ws, size_t ws_bytes,
                                               void* stream) {
  TFRS_CHECK_ARG(q && c && lse && dq && dc && B > 0 && H > 0 && C >= B && d > 0, "inbatch_softmax_maxsim_bwd: bad arguments");
  TFRS_CHECK_ARG(C < (1ll << 31) && B * H < (1ll << 31), "inbatch_softmax_maxsim_bwd: B*H / C too large");
  if (!ws || ws_bytes < tfrs_inbatch_softmax_maxsim_workspace_bytes(B, H, C, d)) { set_error("inbatch_softmax_maxsim: workspace too small"); return TFRS_ERR_WORKSPACE_TOO_SMALL; }
  cudaStream_t st = (cudaStream_t)stream;
  const long long Rq = smx_queries_per_block(B, H, C);
  float* S = (float*)ws;
  float* part = (float*)((unsigned char*)ws + align_up((size_t)Rq * H * C * 4, 256) + align_up((size_t)B * 4, 256));
  for (long long q0 = 0; q0 < B; q0 += Rq) {
    const int nq = (int)((B - q0) < Rq ? (B - q0) : Rq);
    const int rows = nq * H;
    const float* qb = q + q0 * H * d;
    int rc = launch_sgemm<false, true>(qb, d, c, d, rows, (int)C, d, 1, EpiStore{S, C}, st);
    if (rc) return rc;
    sm_make_grad_maxsim<<<(unsigned)nq, SM_THREADS, 0, st>>>(S, C, (int)C, H, q0, inv_temperature, sample_weight, lse, grad_loss);
    TFRS_LAUNCH_CHECK();
    rc = launch_sgemm_split_k<false, false>(S, C, c, d, rows, d, (int)C, SM_DQ_SPLITS, part, dq + q0 * H * d, st);
    if (rc) return rc;
    rc = launch_sgemm<true, false>(S, C, qb, d, (int)C, d, rows, 1, EpiAccum{dc, d, q0 > 0}, st);
    if (rc) return rc;
  }
  return TFRS_OK;
}
