// hardneg.cu -- hard-negative mining inside the Retrieval loss without the [B,C] logits
//   tasks/retrieval.py:205-210 + layers/loss.py:61-111:  top_k(logits + labels * MAX_FLOAT, n + 1) keeps the positive and
//   the n highest-scoring negatives of every query; the loss is the softmax cross-entropy over those n + 1 logits.
// The n + 1 best candidates of every query come from the brute-force scan (tfrs_topk_tc_f32 / tfrs_topk_scan_f32: exact
// fp32 scores, (score desc, index asc) order) -- "hard negatives = a top-K problem".  From that list this file
//   forward : drops the positive if the list holds it (else the list's last entry), soft-maxes {positive} U {n negatives}
//             with the temperature, writes the weighted row loss and the gradient coefficients
//   backward: dq_i = sum_t coef_it c_{j_t} (one warp per query, fixed order);  dc_j += coef_it q_i (red.global.add.f32).
// A positive temperature keeps the order of the scores, so selecting on s instead of s / T picks the same set (up to
// exact fp32 ties created by the division, which have identical logits and therefore the same loss).
#include "common.cuh"

namespace tfrs {

// coef layout per row: [0, k1) coefficient of list entry t (0 for the dropped entry), [k1] coefficient of the positive
// (its probability - 1), [k1 + 1] the weighted row loss.  Coefficients already carry w_i / T.
__global__ void __launch_bounds__(256)
hardneg_fwd_kernel(const float* __restrict__ top_s, const long long* __restrict__ top_i, long long B, int k1,
                   const float* __restrict__ pos, float inv_t, const float* __restrict__ w, float* __restrict__ coef) {
  const int lane = threadIdx.x & 31;
  const long long row = ((long long)blockIdx.x * 256 + threadIdx.x) >> 5;
  if (row >= B) return;
  const float* s = top_s + row * k1;
  const long long* id = top_i + row * k1;
  float* cf = coef + row * (k1 + 2);
  // the positive is candidate `row` (labels = eye, retrieval.py:185): drop it from the negatives if the list holds it
  int drop = k1 - 1;
  for (int t0 = 0; t0 < k1; t0 += 32) {
    const int t = t0 + lane;
    const unsigned hit = __ballot_sync(0xffffffffu, t < k1 && id[t] == row);
    if (hit) { drop = t0 + __ffs(hit) - 1; break; }
  }
  const float lp = pos[row] * inv_t;
  float m = lp;
  for (int t = lane; t < k1; t += 32)
    if (t != drop) m = fmaxf(m, s[t] * inv_t);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  float z = 0.f;
  for (int t = lane; t < k1; t += 32)
    if (t != drop) z += expf(s[t] * inv_t - m);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) z += __shfl_xor_sync(0xffffffffu, z, o);
  const float ep = expf(lp - m);
  z += ep;
  const float wi = w ? w[row] : 1.0f;
  const float g = wi * inv_t / z;
  for (int t = lane; t < k1; t += 32) cf[t] = (t != drop) ? expf(s[t] * inv_t - m) * g : 0.f;
  if (lane == 0) {
    cf[k1] = (ep / z - 1.0f) * wi * inv_t;
    cf[k1 + 1] = wi * ((m - lp) + logf(z));   // lse - positive
  }
}

// one warp per query: dq_i (registers, fixed order) and the scattered dc contributions
__global__ void __launch_bounds__(256)
hardneg_bwd_kernel(const float* __restrict__ q, const float* __restrict__ c, long long B, int d,
                   const long long* __restrict__ top_i, int k1, const float* __restrict__ coef,
                   const float* __restrict__ grad_loss, float* __restrict__ dq, float* __restrict__ dc) {
  const int lane = threadIdx.x & 31;
  const long long row = ((long long)blockIdx.x * 256 + threadIdx.x) >> 5;
  if (row >= B) return;
  const float gl = grad_loss ? grad_loss[0] : 1.0f;
  const long long* id = top_i + row * k1;
  const float* cf = coef + row * (k1 + 2);
  for (int c0 = 0; c0 < d; c0 += 32) {       // 32 columns at a time (d = 64 -> two sweeps over the list, L1/L2 hits)
    const int col = c0 + lane;
    const bool ok = col < d;
    const float qv = ok ? q[row * d + col] : 0.f;
    float acc = 0.f;
    for (int t = 0; t <= k1; ++t) {
      const float a = cf[t] * gl;
      if (a == 0.f) continue;                 // warp-uniform (the dropped entry)
      const long long j = t < k1 ? id[t] : row;
      if (ok) {
        acc = fmaf(a, __ldg(c + j * d + col), acc);
        atomicAdd(dc + j * d + col, a * qv);
      }
    }
    if (ok) dq[row * d + col] = acc;
  }
}

}  // namespace tfrs
using namespace tfrs;

extern "C" int tfrs_hardneg_loss_fwd(const float* top_scores, const int64_t* top_idx, int64_t B, int k1, const float* positive_scores,
                                     float inv_temperature, const float* sample_weight, float* loss, float* coef, void* stream) {
  TFRS_CHECK_ARG(top_scores && top_idx && positive_scores && loss && coef, "hardneg_loss_fwd: NULL pointer");
  TFRS_CHECK_ARG(B > 0 && k1 >= 1, "hardneg_loss_fwd: bad shape");
  TFRS_CHECK_ARG(inv_temperature > 0.f, "hardneg_loss_fwd: needs a positive temperature");
  cudaStream_t st = (cudaStream_t)stream;
  hardneg_fwd_kernel<<<(unsigned)ceil_div(B * 32, 256), 256, 0, st>>>(top_scores, (const long long*)top_idx, B, k1, positive_scores,
                                                                       inv_temperature, sample_weight, coef);
  TFRS_LAUNCH_CHECK();
  return reduce_loss(coef + k1 + 1, B, k1 + 2, loss, st);   // the row losses, fixed order, fp64
}

extern "C" int tfrs_hardneg_loss_bwd(const float* q, const float* c, int64_t B, int64_t C, int d, const int64_t* top_idx, int k1,
                                     const float* coef, const float* grad_loss, float* dq, float* dc, void* stream) {
  TFRS_CHECK_ARG(q && c && top_idx && coef && dq && dc, "hardneg_loss_bwd: NULL pointer");
  TFRS_CHECK_ARG(B > 0 && C >= B && d > 0 && k1 >= 1, "hardneg_loss_bwd: bad shape");
  cudaStream_t st = (cudaStream_t)stream;
  TFRS_CUDA(cudaMemsetAsync(dc, 0, (size_t)C * d * sizeof(float), st));
  hardneg_bwd_kernel<<<(unsigned)ceil_div(B * 32, 256), 256, 0, st>>>(q, c, B, d, (const long long*)top_idx, k1, coef, grad_loss, dq, dc);
  TFRS_LAUNCH_CHECK();
  return TFRS_OK;
}
