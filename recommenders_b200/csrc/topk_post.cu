// topk_post.cu -- the small per-query steps AFTER a top-K list exists, for the paths that do not go through the
// tensor-core finalize (small corpora, Streaming's carried state, lists merged across shards):
//   tfrs_topk_exclude_rerank_f32 : `_exclude` (layers/factorized_top_k.py:83-115) on an over-fetched [Q, kf] list
//   tfrs_count_above_f32         : #{retrieved scores > positive score}   (metrics/factorized_top_k.py:181-192, in_top_k)
//   tfrs_topk_hits_accumulate    : the weighted running sums behind FactorizedTopK's Mean metrics, kept on the device
// One warp per query, no atomics, deterministic.  An array with no elements may be NULL (torch hands out a NULL
// data_ptr for empty tensors): exclusions when n_excl == 0, scores when k == 0, every per-query array when Q == 0.
#include "common.cuh"

namespace tfrs {

__device__ __forceinline__ unsigned int okey(float f) {  // larger float <=> larger unsigned; -0 canonicalised by the caller
  unsigned int u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

constexpr int XR_THREADS = 128;

__global__ void __launch_bounds__(XR_THREADS)
exclude_rerank_kernel(const float* __restrict__ scores, const long long* __restrict__ idx, long long Q, int kf,
                      const long long* __restrict__ identifiers, const long long* __restrict__ exclusions, int n_excl,
                      int k_out, int warps, float* __restrict__ out_s, long long* __restrict__ out_i) {
  extern __shared__ __align__(16) unsigned char xsm[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (warp >= warps) return;
  const long long row = (long long)blockIdx.x * warps + warp;
  if (row >= Q) return;
  unsigned long long* akey = reinterpret_cast<unsigned long long*>(xsm) + (size_t)warp * kf;
  const float* s = scores + row * kf;
  const long long* ix = idx + row * kf;
  for (int t = lane; t < kf; t += 32) {
    const long long gi = ix[t];
    const long long ident = identifiers ? __ldg(identifiers + gi) : gi;
    bool isin = false;
    for (int x = 0; x < n_excl; ++x) isin |= (__ldg(exclusions + row * n_excl + x) == ident);
    const float adj = (isin ? s[t] - 1.0e5f : s[t]) + 0.0f;   // scores - isin * 1e5 (:104-107)
    akey[t] = ((unsigned long long)okey(adj) << 32) | (unsigned long long)(0xFFFFFFFFu - (unsigned int)t);
  }
  __syncwarp();
  for (int t = lane; t < kf; t += 32) {   // top_k(adjusted, k): ties -> lower position; outputs are the ORIGINAL entries
    const unsigned long long mine = akey[t];
    int rank = 0;
    for (int j = 0; j < kf; ++j) rank += (akey[j] > mine) ? 1 : 0;
    if (rank < k_out) { out_s[row * k_out + rank] = s[t]; out_i[row * k_out + rank] = ix[t]; }
  }
}

__global__ void __launch_bounds__(256)
count_above_kernel(const float* __restrict__ scores, long long ld, int k, const float* __restrict__ pos, long long Q,
                   int* __restrict__ out_count) {
  const int lane = threadIdx.x & 31;
  const long long row = ((long long)blockIdx.x * 256 + threadIdx.x) >> 5;
  if (row >= Q) return;
  const float p = pos[row];
  int c = 0;
  for (int t = lane; t < k; t += 32) c += (scores[row * ld + t] > p) ? 1 : 0;   // NaN padding compares false
  c = __reduce_add_sync(0xffffffffu, c);
  if (lane == 0) out_count[row] = c;
}

constexpr int HA_MAX_KS = 16;
struct HitParams { int ks[HA_MAX_KS]; int n_ks; };

// acc[j] += sum_i w_i * [count_i < ks[j] and pos_i finite]   (j < n_ks);   acc[n_ks] += sum_i w_i  (w = 1 without weights)
// One CTA, fixed-order fp64 tree: deterministic.
__global__ void __launch_bounds__(256)
hits_accumulate_kernel(const int* __restrict__ count, const float* __restrict__ pos, const float* __restrict__ weight,
                       long long Q, HitParams hp, double* __restrict__ acc) {
  __shared__ double red[256];
  for (int j = 0; j <= hp.n_ks; ++j) {
    double a = 0.0;
    for (long long i = threadIdx.x; i < Q; i += 256) {
      const double w = weight ? (double)weight[i] : 1.0;
      if (j == hp.n_ks) a += w;
      else if (count[i] < hp.ks[j] && isfinite(pos[i])) a += w;
    }
    red[threadIdx.x] = a;
    __syncthreads();
    for (int o = 128; o > 0; o >>= 1) { if (threadIdx.x < o) red[threadIdx.x] += red[threadIdx.x + o]; __syncthreads(); }
    if (threadIdx.x == 0) acc[j] += red[0];
    __syncthreads();
  }
}

}  // namespace tfrs
using namespace tfrs;

extern "C" int tfrs_topk_exclude_rerank_f32(const float* scores, const int64_t* idx, int64_t Q, int k_fetched,
                                            const int64_t* identifiers, const int64_t* exclusions, int n_excl, int k_out,
                                            float* out_scores, int64_t* out_idx, void* stream) {
  TFRS_CHECK_ARG(scores && idx && (exclusions || n_excl == 0) && out_scores && out_idx, "exclude_rerank: NULL pointer");
  TFRS_CHECK_ARG(Q >= 0 && k_fetched > 0 && k_fetched <= 4096 && n_excl >= 0 && k_out > 0 && k_out <= k_fetched,
                 "exclude_rerank: bad shape (k_fetched=%d k_out=%d)", k_fetched, k_out);
  if (Q == 0) return TFRS_OK;
  const int warps = k_fetched <= 1024 ? XR_THREADS / 32 : 1;
  const size_t smem = (size_t)warps * k_fetched * 8;
  TFRS_DYN_SMEM(exclude_rerank_kernel, 64 * 1024);
  exclude_rerank_kernel<<<(unsigned)ceil_div(Q, warps), XR_THREADS, smem, (cudaStream_t)stream>>>(
      scores, (const long long*)idx, Q, k_fetched, (const long long*)identifiers, (const long long*)exclusions, n_excl, k_out,
      warps, out_scores, (long long*)out_idx);
  TFRS_LAUNCH_CHECK();
  return TFRS_OK;
}

extern "C" int tfrs_count_above_f32(const float* scores, int64_t ld, int k, const float* positive_scores, int64_t Q,
                                    int32_t* out_count, void* stream) {
  TFRS_CHECK_ARG((Q <= 0 || ((scores || k == 0) && positive_scores && out_count)) && ld >= k && k >= 0,
                 "count_above: bad argument");
  if (Q <= 0) return TFRS_OK;
  count_above_kernel<<<(unsigned)ceil_div(Q * 32, 256), 256, 0, (cudaStream_t)stream>>>(scores, ld, k, positive_scores, Q, out_count);
  TFRS_LAUNCH_CHECK();
  return TFRS_OK;
}

extern "C" int tfrs_topk_hits_accumulate(const int32_t* count, const float* positive_scores, const float* sample_weight, int64_t Q,
                                         const int32_t* ks, int n_ks, double* acc, void* stream) {
  TFRS_CHECK_ARG(((count && positive_scores) || Q <= 0) && ks && acc && n_ks > 0 && n_ks <= HA_MAX_KS,
                 "hits_accumulate: bad argument (n_ks <= 16)");
  if (Q <= 0) return TFRS_OK;
  HitParams hp{};
  hp.n_ks = n_ks;
  for (int j = 0; j < n_ks; ++j) hp.ks[j] = ks[j];   // ks is a HOST array
  hits_accumulate_kernel<<<1, 256, 0, (cudaStream_t)stream>>>(count, positive_scores, sample_weight, Q, hp, acc);
  TFRS_LAUNCH_CHECK();
  return TFRS_OK;
}
