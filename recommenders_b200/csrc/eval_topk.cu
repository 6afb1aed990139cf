// eval_topk.cu -- K14: exact top-K where each query lists rows that score exactly -1e6 instead of their dot, and the
// hit count over those top-K rows; the device side of examples.movielens.evaluate (examples/movielens.py:71-88:
// `scores[train_movies] = -1e6`, `top_movies = argsort(-scores)[:k]`, `sum(x in top_movies for x in test_movies)`).
//
//   tfrs_topk_override_merge_f32   scan route: the query's top-w list by true score (w >= min(N, k + e), e = the listed
//                                  rows) -> drop the listed rows (binary search in the query's sorted list) -> merge the
//                                  first k survivors with the listed rows at -1e6 in row order -> k.  One warp per query.
//   tfrs_topk_overriding_dense_f32 dense route, any list length: per chunk of queries gather the query rows, score the
//                                  chunk with the exact SGEMM (sgemm.cuh), write -1e6 over the listed entries, select
//                                  the top k per row with rowselect.cuh, scatter the rows to their queries.
//   tfrs_count_listed              hits: one warp per query, its k rows in shared memory, one search per CSR entry.
// Lists are CSR: offsets int64 [Q+1], rows int64.  Order = (score desc, row asc) everywhere, so both routes give the
// same bits.
#include "rowselect.cuh"
#include "sgemm.cuh"

namespace tfrs {

constexpr float OVERRIDE_SCORE = -1.0e6f;
constexpr int OM_WARPS = 4;          // queries per CTA of the merge and count kernels
constexpr int OM_MAX_K = 256;        // the scan route's k <= w <= TC_MAX_K

// first position p in sorted a[0, n) with a[p] >= x
__device__ __forceinline__ int lower_bound_i64(const long long* a, int n, long long x) {
  int lo = 0, hi = n;
  while (lo < hi) { const int mid = (lo + hi) >> 1; if (a[mid] < x) lo = mid + 1; else hi = mid; }
  return lo;
}

__global__ void __launch_bounds__(OM_WARPS * 32)
override_merge_kernel(const float* __restrict__ ls, const long long* __restrict__ li, int w, long long n,
                      const long long* __restrict__ users, const long long* __restrict__ offsets,
                      const long long* __restrict__ rows, int k, int k_out, float* __restrict__ out_s,
                      long long* __restrict__ out_i, int out_ld) {
  __shared__ float ss[OM_WARPS][OM_MAX_K];
  __shared__ long long si[OM_WARPS][OM_MAX_K];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long j = (long long)blockIdx.x * OM_WARPS + warp;
  if (j >= n) return;
  const long long u = users ? users[j] : j;
  const long long* L = rows + offsets[u];
  const long long e = offsets[u + 1] - offsets[u];
  float* s_sh = ss[warp];
  long long* i_sh = si[warp];

  // survivors: the list's rows that are not listed, in list order (= the total order), the first k of them
  int ns = 0;
  for (int base = 0; base < w && ns < k; base += 32) {
    const int t = base + lane;
    bool surv = false;
    float s = 0.f; long long i = 0;
    if (t < w) {
      s = ls[j * w + t]; i = li[j * w + t];
      const int p = lower_bound_i64(L, (int)e, i);
      surv = !(p < e && L[p] == i);
    }
    const unsigned m = __ballot_sync(0xffffffffu, surv);
    const int r = ns + __popc(m & ((1u << lane) - 1u));
    if (surv && r < k) { s_sh[r] = s; i_sh[r] = i; }
    ns += __popc(m);
  }
  ns = ns < k ? ns : k;
  __syncwarp();

  // Only the first min(e, k) listed rows can reach the output: they all score -1e6 and are ordered by row.
  const int ne = (int)(e < k ? e : k);
  for (int r = lane; r < ns; r += 32) {   // survivor r: r survivors and the listed rows that precede it come first
    const float s = s_sh[r]; const long long i = i_sh[r];
    const int before = (OVERRIDE_SCORE > s) ? ne : (OVERRIDE_SCORE == s ? lower_bound_i64(L, ne, i) : 0);
    const int rank = r + before;
    if (rank < k_out) { out_s[u * out_ld + rank] = s; out_i[u * out_ld + rank] = i; }
  }
  for (int x = lane; x < ne; x += 32) {   // listed row x: x listed rows and the survivors that precede it come first
    const long long l = L[x];
    int lo = 0, hi = ns;
    while (lo < hi) { const int mid = (lo + hi) >> 1; if (better(s_sh[mid], i_sh[mid], OVERRIDE_SCORE, l)) lo = mid + 1; else hi = mid; }
    const int rank = x + lo;
    if (rank < k_out) { out_s[u * out_ld + rank] = OVERRIDE_SCORE; out_i[u * out_ld + rank] = l; }
  }
}

// ---- dense route -------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
gather_queries_kernel(const float* __restrict__ q, int d, const long long* __restrict__ users, long long u0, int c,
                      float* __restrict__ qc) {
  const long long n = (long long)c * d;
  for (long long t = (long long)blockIdx.x * 256 + threadIdx.x; t < n; t += (long long)gridDim.x * 256) {
    const long long r = t / d, col = t - r * d;
    const long long u = users ? users[u0 + r] : u0 + r;
    qc[t] = q[u * d + col];
  }
}

// one CTA per row of the chunk: S[r, listed] = -1e6
__global__ void __launch_bounds__(256)
override_scores_kernel(float* __restrict__ S, long long N, const long long* __restrict__ users, long long u0,
                       const long long* __restrict__ offsets, const long long* __restrict__ rows) {
  const long long r = blockIdx.x;
  const long long u = users ? users[u0 + r] : u0 + r;
  const long long b = offsets[u], end = offsets[u + 1];
  for (long long t = b + threadIdx.x; t < end; t += 256) S[r * N + rows[t]] = OVERRIDE_SCORE;
}

struct ChunkRowProvider {   // row r of the score chunk; the index is the corpus row
  const float* S; long long N;
  __device__ void begin(int, void*) {}
  __device__ long long count(int) const { return N; }
  __device__ void get(int row, long long t, float& s, long long& i) const { s = S[(long long)row * N + t]; i = t; }
};

__global__ void __launch_bounds__(256)
scatter_rows_kernel(const float* __restrict__ ts, const long long* __restrict__ ti, int c, int k_out,
                    const long long* __restrict__ users, long long u0, float* __restrict__ out_s,
                    long long* __restrict__ out_i, int out_ld) {
  const long long n = (long long)c * k_out;
  for (long long t = (long long)blockIdx.x * 256 + threadIdx.x; t < n; t += (long long)gridDim.x * 256) {
    const long long r = t / k_out, col = t - r * k_out;
    const long long u = users ? users[u0 + r] : u0 + r;
    out_s[u * out_ld + col] = ts[t]; out_i[u * out_ld + col] = ti[t];
  }
}

struct DensePlan { long long chunk; size_t q_bytes, s_bytes, t_bytes; };

static size_t dense_bytes(long long c, long long N, int d, int k_out, DensePlan* p) {
  const size_t qb = align_up((size_t)c * d * 4, 256), sb = align_up((size_t)c * N * 4, 256),
               tb = align_up((size_t)c * k_out * 4, 256) + align_up((size_t)c * k_out * 8, 256);
  if (p) { p->chunk = c; p->q_bytes = qb; p->s_bytes = sb; p->t_bytes = tb; }
  return qb + sb + tb;
}

constexpr size_t DENSE_CHUNK_BUDGET = (size_t)256 << 20;   // bytes of one chunk's workspace by default

// ---- hits ---------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(OM_WARPS * 32)
count_listed_kernel(const long long* __restrict__ top, long long Q, int kk, long long ld,
                    const long long* __restrict__ offsets, const long long* __restrict__ rows, int* __restrict__ out) {
  extern __shared__ __align__(16) unsigned char cl_smem[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long q = (long long)blockIdx.x * OM_WARPS + warp;
  if (q >= Q) return;
  long long* t_sh = reinterpret_cast<long long*>(cl_smem) + (size_t)warp * kk;
  for (int t = lane; t < kk; t += 32) t_sh[t] = top[q * ld + t];
  __syncwarp();
  int c = 0;
  for (long long t = offsets[q] + lane; t < offsets[q + 1]; t += 32) {
    const long long x = rows[t];
    bool hit = false;
    for (int j = 0; j < kk && !hit; ++j) hit = (t_sh[j] == x);
    c += hit ? 1 : 0;
  }
  c = __reduce_add_sync(0xffffffffu, c);
  if (lane == 0) out[q] = c;
}

}  // namespace tfrs

using namespace tfrs;

extern "C" int tfrs_topk_override_merge_f32(const float* list_scores, const int64_t* list_idx, int64_t n, int w,
                                            const int64_t* users, const int64_t* offsets, const int64_t* rows, int k,
                                            int k_out, float* out_scores, int64_t* out_idx, int out_ld, void* stream) {
  TFRS_CHECK_ARG(n >= 0 && k > 0 && w >= k_out && w <= OM_MAX_K && k_out > 0 && k_out <= k && out_ld >= k_out,
                 "topk_override_merge: bad shape (w=%d k=%d k_out=%d out_ld=%d; k_out <= k, k_out <= w <= %d)", w, k,
                 k_out, out_ld, OM_MAX_K);
  if (n == 0) return TFRS_OK;
  TFRS_CHECK_ARG(list_scores && list_idx && offsets && out_scores && out_idx, "topk_override_merge: NULL pointer");
  override_merge_kernel<<<(unsigned)ceil_div(n, OM_WARPS), OM_WARPS * 32, 0, (cudaStream_t)stream>>>(
      list_scores, (const long long*)list_idx, w, n, (const long long*)users, (const long long*)offsets,
      (const long long*)rows, k, k_out, out_scores, (long long*)out_idx, out_ld);
  TFRS_LAUNCH_CHECK();
  return TFRS_OK;
}

extern "C" size_t tfrs_topk_overriding_dense_workspace_bytes(int64_t n, int64_t N, int d, int k) {
  if (n <= 0 || N <= 0 || d <= 0 || k <= 0) return 256;
  const int k_out = (int)(k < N ? k : N);
  const size_t per = dense_bytes(1, N, d, k_out, nullptr);
  long long c = (long long)(DENSE_CHUNK_BUDGET / per);
  if (c < 1) c = 1;
  if (c > n) c = n;
  return dense_bytes(c, N, d, k_out, nullptr);
}

extern "C" int tfrs_topk_overriding_dense_f32(const float* q, const int64_t* users, int64_t n, const float* corpus,
                                              int64_t N, int d, int k, const int64_t* offsets, const int64_t* rows,
                                              float* out_scores, int64_t* out_idx, int out_ld, void* ws, size_t ws_bytes,
                                              void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  TFRS_CHECK_ARG(n >= 0 && N >= 0 && d > 0 && k > 0 && k <= 2048, "topk_overriding_dense: bad shape n=%lld N=%lld d=%d k=%d",
                 (long long)n, (long long)N, d, k);
  TFRS_CHECK_ARG(N < (1ll << 31), "topk_overriding_dense: N must be < 2^31");
  if (n == 0 || N == 0) return TFRS_OK;
  const int k_out = (int)(k < N ? k : N);
  TFRS_CHECK_ARG(out_ld >= k_out, "topk_overriding_dense: out_ld=%d < %d", out_ld, k_out);
  TFRS_CHECK_ARG(q && corpus && offsets && out_scores && out_idx, "topk_overriding_dense: NULL pointer");
  // the largest chunk the workspace holds
  DensePlan plan;
  long long c = (long long)(ws_bytes / dense_bytes(1, N, d, k_out, nullptr));
  if (c > n) c = n;
  while (c > 0 && dense_bytes(c, N, d, k_out, &plan) > ws_bytes) --c;
  if (!ws || c < 1) {
    set_error("topk_overriding_dense: workspace too small (%zu < %zu)", ws_bytes, dense_bytes(1, N, d, k_out, nullptr));
    return TFRS_ERR_WORKSPACE_TOO_SMALL;
  }
  TFRS_CHECK_ARG(c < 65536ll * SG_BM, "topk_overriding_dense: chunk too large");
  unsigned char* p = (unsigned char*)ws;
  float* qc = (float*)p; p += plan.q_bytes;
  float* S = (float*)p; p += plan.s_bytes;
  float* ts = (float*)p; p += align_up((size_t)c * k_out * 4, 256);
  long long* ti = (long long*)p;

  const int cap = rowselect_cap(k_out);
  const size_t smem = rowselect_smem(cap, 0);
  TFRS_DYN_SMEM(row_topk_kernel<ChunkRowProvider>, 64 * 1024);
  for (long long u0 = 0; u0 < n; u0 += c) {
    const int cc = (int)(n - u0 < c ? n - u0 : c);
    gather_queries_kernel<<<elementwise_grid((long long)cc * d), 256, 0, st>>>(q, d, (const long long*)users, u0, cc, qc);
    TFRS_LAUNCH_CHECK();
    int rc = launch_sgemm<false, true>(qc, d, corpus, d, cc, (int)N, d, 1, EpiStore{S, N}, st);
    if (rc) return rc;
    override_scores_kernel<<<(unsigned)cc, 256, 0, st>>>(S, N, (const long long*)users, u0, (const long long*)offsets,
                                                         (const long long*)rows);
    TFRS_LAUNCH_CHECK();
    row_topk_kernel<ChunkRowProvider><<<(unsigned)cc, RS_THREADS, smem, st>>>(ChunkRowProvider{S, N}, k_out, cap, ts, ti, k_out);
    TFRS_LAUNCH_CHECK();
    scatter_rows_kernel<<<elementwise_grid((long long)cc * k_out), 256, 0, st>>>(ts, ti, cc, k_out, (const long long*)users, u0,
                                                                                 out_scores, (long long*)out_idx, out_ld);
    TFRS_LAUNCH_CHECK();
  }
  return TFRS_OK;
}

extern "C" int tfrs_count_listed(const int64_t* top_rows, int64_t Q, int kk, int64_t ld, const int64_t* offsets,
                                 const int64_t* rows, int32_t* out_count, void* stream) {
  TFRS_CHECK_ARG(Q >= 0 && kk >= 0 && kk <= 2048 && ld >= kk, "count_listed: bad shape (kk=%d ld=%lld; kk <= 2048)", kk,
                 (long long)ld);
  if (Q == 0) return TFRS_OK;
  TFRS_CHECK_ARG((top_rows || kk == 0) && offsets && out_count, "count_listed: NULL pointer");
  const size_t smem = (size_t)OM_WARPS * kk * 8;
  TFRS_DYN_SMEM(count_listed_kernel, 64 * 1024);
  count_listed_kernel<<<(unsigned)ceil_div(Q, OM_WARPS), OM_WARPS * 32, smem, (cudaStream_t)stream>>>(
      (const long long*)top_rows, Q, kk, ld, (const long long*)offsets, (const long long*)rows, out_count);
  TFRS_LAUNCH_CHECK();
  return TFRS_OK;
}
