// dot_interaction.cu -- DLRM pairwise feature interaction (layers/feature_interaction/dot_interaction.py:53-104):
//   feats [B, F, d]  ->  xact[b, i, j] = e_bi . e_bj ; the strictly-lower (or lower incl. diagonal) triangle in
//   row-major (i, j) order [B, F(F-1)/2 | F(F+1)/2], or the full [B, F*F] with the excluded part zeroed (skip_gather).
// HBM-bound (read B*F*d*4, write B*out_dim*4): one warp per sample, the sample's F x d block staged in shared memory
// (row pitch d+1: conflict-free when lanes read different features), every output one sequential fmaf chain
// (the repo's canonical dot product).  Backward: dE_bi = sum_j G'(i,j) e_bj with G' the symmetrised upstream
// gradient (the diagonal counts twice), j ascending -- deterministic.
#include "common.cuh"

namespace tfrs {

constexpr int DI_WARPS = 4;
constexpr int DI_MAX_F = 64;

__device__ __forceinline__ int di_index(int i, int j, int F, bool self, bool skip) {  // position of the (i, j), j <= i, entry
  if (skip) return i * F + j;
  return self ? (i * (i + 1)) / 2 + j : (i * (i - 1)) / 2 + j;
}

__global__ void __launch_bounds__(DI_WARPS * 32)
dot_interaction_fwd_kernel(const float* __restrict__ feats, long long B, int F, int d, bool self, bool skip, int out_dim,
                           float* __restrict__ out) {
  extern __shared__ float di_smem[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int pitch = d + 1;
  float* e = di_smem + (size_t)warp * F * pitch;
  const long long b = (long long)blockIdx.x * DI_WARPS + warp;
  if (b >= B) return;
  const float* src = feats + b * F * d;
  for (int t = lane; t < F * d; t += 32) e[(t / d) * pitch + (t % d)] = src[t];
  __syncwarp();
  float* dst = out + b * out_dim;
  if (skip) {
    for (int p = lane; p < F * F; p += 32) {
      const int i = p / F, j = p - i * F;
      float acc = 0.f;
      if (j < i || (self && j == i)) {
        const float* ei = e + i * pitch; const float* ej = e + j * pitch;
        for (int k = 0; k < d; ++k) acc = fmaf(ei[k], ej[k], acc);
      }
      dst[p] = acc;
    }
  } else {
    // entries in (i, j) row-major order of the lower triangle: walk rows, lanes take consecutive entries
    for (int p = lane; p < out_dim; p += 32) {
      // invert p -> (i, j): i = largest with tri(i) <= p
      int i = (int)((sqrtf(8.0f * (float)p + 1.0f) - 1.0f) * 0.5f);
      if (self) { while ((i + 1) * (i + 2) / 2 <= p) ++i; while (i * (i + 1) / 2 > p) --i; }
      else { i += 1; while ((i + 1) * i / 2 <= p) ++i; while (i * (i - 1) / 2 > p) --i; }
      const int j = p - (self ? i * (i + 1) / 2 : i * (i - 1) / 2);
      const float* ei = e + i * pitch; const float* ej = e + j * pitch;
      float acc = 0.f;
      for (int k = 0; k < d; ++k) acc = fmaf(ei[k], ej[k], acc);
      dst[p] = acc;
    }
  }
}

__global__ void __launch_bounds__(DI_WARPS * 32)
dot_interaction_bwd_kernel(const float* __restrict__ feats, const float* __restrict__ gout, long long B, int F, int d, bool self,
                           bool skip, int out_dim, float* __restrict__ dfeats) {
  extern __shared__ float di_smem[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int pitch = d + 1;
  float* e = di_smem + (size_t)warp * (F * pitch + out_dim);
  float* g = e + F * pitch;
  const long long b = (long long)blockIdx.x * DI_WARPS + warp;
  if (b >= B) return;
  const float* src = feats + b * F * d;
  for (int t = lane; t < F * d; t += 32) e[(t / d) * pitch + (t % d)] = src[t];
  const float* gs = gout + b * out_dim;
  for (int t = lane; t < out_dim; t += 32) g[t] = gs[t];
  __syncwarp();
  float* dst = dfeats + b * F * d;
  for (int t = lane; t < F * d; t += 32) {
    const int i = t / d, k = t - i * d;
    float acc = 0.f;
    for (int j = 0; j < F; ++j) {
      float coef;
      if (j < i) coef = g[di_index(i, j, F, self, skip)];
      else if (j > i) coef = g[di_index(j, i, F, self, skip)];
      else coef = self ? 2.0f * g[di_index(i, i, F, self, skip)] : 0.f;
      acc = fmaf(coef, e[j * pitch + k], acc);
    }
    dst[t] = acc;
  }
}

static int di_out_dim(int F, int self, int skip) { return skip ? F * F : (self ? F * (F + 1) / 2 : F * (F - 1) / 2); }

}  // namespace tfrs
using namespace tfrs;

extern "C" int tfrs_dot_interaction_out_dim(int F, int self_interaction, int skip_gather) {
  return F > 0 ? di_out_dim(F, self_interaction, skip_gather) : 0;
}

static int di_check(const float* feats, int64_t B, int F, int d) {
  TFRS_CHECK_ARG((feats || B == 0) && B >= 0 && F > 0 && d > 0, "dot_interaction: bad arguments");  // empty batch: NULL
  if (F > DI_MAX_F || (size_t)DI_WARPS * (F * (d + 1) + F * F) * 4 > 200 * 1024) {
    set_error("dot_interaction: F=%d, d=%d outside the shared-memory staging range (F <= %d)", F, d, DI_MAX_F);
    return TFRS_ERR_UNSUPPORTED;
  }
  return TFRS_OK;
}

extern "C" int tfrs_dot_interaction_fwd_f32(const float* feats, int64_t B, int F, int d, int self_interaction, int skip_gather,
                                            float* out, void* stream) {
  int rc = di_check(feats, B, F, d);
  if (rc) return rc;
  const int od = di_out_dim(F, self_interaction, skip_gather);
  if (B == 0 || od == 0) return TFRS_OK;  // nothing to write (a single feature without self-interaction has no pairs)
  TFRS_CHECK_ARG(out, "dot_interaction_fwd: NULL output");
  const size_t smem = (size_t)DI_WARPS * F * (d + 1) * 4;
  TFRS_DYN_SMEM(dot_interaction_fwd_kernel, 200 * 1024);
  dot_interaction_fwd_kernel<<<(unsigned)ceil_div(B, DI_WARPS), DI_WARPS * 32, smem, (cudaStream_t)stream>>>(
      feats, B, F, d, self_interaction != 0, skip_gather != 0, od, out);
  TFRS_LAUNCH_CHECK();
  return TFRS_OK;
}

extern "C" int tfrs_dot_interaction_bwd_f32(const float* feats, const float* gout, int64_t B, int F, int d, int self_interaction,
                                            int skip_gather, float* dfeats, void* stream) {
  int rc = di_check(feats, B, F, d);
  if (rc) return rc;
  if (B == 0) return TFRS_OK;
  const int od = di_out_dim(F, self_interaction, skip_gather);
  // a single feature without self-interaction has no outputs: its upstream gradient is empty (NULL) and dE is zero
  TFRS_CHECK_ARG(dfeats && (gout || od == 0), "dot_interaction_bwd: NULL pointer");
  const size_t smem = (size_t)DI_WARPS * (F * (d + 1) + od) * 4;
  TFRS_DYN_SMEM(dot_interaction_bwd_kernel, 200 * 1024);
  dot_interaction_bwd_kernel<<<(unsigned)ceil_div(B, DI_WARPS), DI_WARPS * 32, smem, (cudaStream_t)stream>>>(
      feats, gout, B, F, d, self_interaction != 0, skip_gather != 0, od, dfeats);
  TFRS_LAUNCH_CHECK();
  return TFRS_OK;
}
