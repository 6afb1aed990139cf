// topk.cu -- exact fp32 brute-force top-K scan (CUDA-core anchor path) and the list merge.
//
//   tfrs_topk_scan_f32 : layers/factorized_top_k.py:603-605 (BruteForce.call) and :424-472
//                        (Streaming's per-chunk top_k + running merge), chunk by chunk:
//                        scores chunk = exact SGEMM (sgemm.cuh) -> per-row select (rowselect.cuh).
//   tfrs_topk_merge_strided : Streaming.reduce (:440-472) / the shard merge after the all-gather.
#include "rowselect.cuh"
#include "sgemm.cuh"

namespace tfrs {

struct ScanProvider {
  const float* st_s; const long long* st_i; int st_k; int st_ld;  // carried state (nullable when st_k == 0)
  const float* S; long long ldS; int nc; long long base;          // scores chunk [Q, nc], index of column 0
  __device__ void begin(int, void*) {}
  __device__ long long count(int) const { return (long long)st_k + nc; }
  __device__ void get(int row, long long t, float& s, long long& i) const {
    if (t < st_k) { s = st_s[(long long)row * st_ld + t]; i = st_i[(long long)row * st_ld + t]; }
    else { long long j = t - st_k; s = __ldg(S + (long long)row * ldS + j); i = base + j; }
  }
};

struct MergeProvider {
  const float* s; const long long* idx; int n_lists; long long Q; int k_in;
  long long stride_s, stride_i;  // elements between consecutive lists
  __device__ void begin(int, void*) {}
  __device__ long long count(int) const { return (long long)n_lists * k_in; }
  __device__ void get(int row, long long t, float& sc, long long& i) const {
    int l = (int)(t / k_in), r = (int)(t % k_in);
    long long o = (long long)row * k_in + r;
    sc = s[(long long)l * stride_s + o]; i = idx[(long long)l * stride_i + o];
  }
};

struct ScanPlan { long long nc; size_t s_bytes; size_t state_bytes; size_t total; };

static ScanPlan scan_plan(long long Q, long long N, int k, size_t budget) {
  ScanPlan p;
  const size_t target = budget ? budget : (size_t)256 << 20;
  p.state_bytes = align_up((size_t)Q * k * 4, 256) + align_up((size_t)Q * k * 8, 256);
  long long n_pad = ceil_div(N > 0 ? N : 1, 128) * 128;
  long long nc = (long long)(target / ((size_t)Q * 4)) / 128 * 128;
  if (nc < 1024) nc = 1024;
  if (nc > n_pad) nc = n_pad;
  p.nc = nc;
  p.s_bytes = align_up((size_t)Q * nc * 4, 256);
  p.total = p.s_bytes + 2 * p.state_bytes;
  return p;
}

template <class Prov>
static int launch_row_topk(Prov prov, long long Q, int k, float* out_s, long long* out_i, int out_ld,
                           cudaStream_t st) {
  int cap = rowselect_cap(k);
  size_t smem = rowselect_smem(cap, 0);
  TFRS_DYN_SMEM(row_topk_kernel<Prov>, 64 * 1024);
  row_topk_kernel<Prov><<<(unsigned)Q, RS_THREADS, smem, st>>>(prov, k, cap, out_s, out_i, out_ld);
  TFRS_LAUNCH_CHECK();
  return TFRS_OK;
}

}  // namespace tfrs

using namespace tfrs;

extern "C" size_t tfrs_topk_scan_workspace_bytes(int64_t Q, int64_t N, int d, int k) {
  (void)d;
  if (Q <= 0 || k <= 0) return 256;
  return scan_plan(Q, N, k, 0).total;
}

extern "C" int tfrs_topk_scan_f32(const float* q, int64_t Q, const float* corpus, int64_t N, int d, int k,
                                  int64_t index_offset, const float* state_scores, const int64_t* state_idx,
                                  int state_k, float* out_scores, int64_t* out_idx, void* ws, size_t ws_bytes,
                                  void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  TFRS_CHECK_ARG(Q >= 0 && N >= 0 && d > 0, "topk_scan: bad shape Q=%lld N=%lld d=%d", (long long)Q, (long long)N, d);
  TFRS_CHECK_ARG(k > 0 && k <= 2048, "topk_scan: k=%d out of range (1..2048)", k);
  TFRS_CHECK_ARG(state_k >= 0 && state_k <= k, "topk_scan: state_k=%d must be in [0,k]", state_k);
  TFRS_CHECK_ARG(state_k == 0 || (state_scores && state_idx), "topk_scan: state pointers are NULL");
  TFRS_CHECK_ARG(Q < (1ll << 31) && N < (1ll << 31), "topk_scan: Q/N must be < 2^31 per call");
  if (Q == 0 || (N == 0 && state_k == 0)) return TFRS_OK;
  TFRS_CHECK_ARG(q && out_scores && out_idx && (N == 0 || corpus), "topk_scan: NULL pointer");

  ScanPlan plan = scan_plan(Q, N, k, 0);
  if (ws_bytes < plan.total) {
    // try to shrink the chunk to what was given
    size_t fixed = 2 * plan.state_bytes;
    if (ws_bytes > fixed + (size_t)Q * 1024 * 4) plan = scan_plan(Q, N, k, ws_bytes - fixed - 256);
    if (!ws || ws_bytes < plan.total) {
      set_error("topk_scan: workspace too small (%zu < %zu)", ws_bytes, plan.total);
      return TFRS_ERR_WORKSPACE_TOO_SMALL;
    }
  }
  unsigned char* w = (unsigned char*)ws;
  float* S = (float*)w; w += plan.s_bytes;
  float* stS[2]; long long* stI[2];
  for (int b = 0; b < 2; ++b) {
    stS[b] = (float*)w; w += align_up((size_t)Q * k * 4, 256);
    stI[b] = (long long*)w; w += align_up((size_t)Q * k * 8, 256);
  }

  const float* cur_s = state_scores; const long long* cur_i = (const long long*)state_idx;
  int cur_k = state_k, cur_ld = state_k;  // the caller's state is dense [Q, state_k]
  if (N == 0) {  // only a state: re-select (sorts it)
    ScanProvider prov{cur_s, cur_i, cur_k, cur_ld, nullptr, 0, 0, 0};
    return launch_row_topk(prov, Q, k, out_scores, (long long*)out_idx, k, st);
  }
  int buf = 0;
  for (long long c0 = 0; c0 < N; c0 += plan.nc) {
    int nc = (int)((N - c0) < plan.nc ? (N - c0) : plan.nc);
    int rc = launch_sgemm<false, true>(q, d, corpus + c0 * d, d, (int)Q, nc, d, 1, EpiStore{S, plan.nc}, st);
    if (rc) return rc;
    bool last = (c0 + plan.nc >= N);
    float* o_s = last ? out_scores : stS[buf];
    long long* o_i = last ? (long long*)out_idx : stI[buf];
    ScanProvider prov{cur_s, cur_i, cur_k, cur_ld, S, plan.nc, nc, index_offset + c0};
    rc = launch_row_topk(prov, Q, k, o_s, o_i, k, st);
    if (rc) return rc;
    long long seen = (long long)cur_k + nc;
    cur_k = (int)(seen < k ? seen : k);
    cur_s = o_s; cur_i = o_i; cur_ld = k;
    buf ^= 1;
  }
  return TFRS_OK;
}

extern "C" int tfrs_topk_merge_strided(const float* scores, const int64_t* idx, int64_t list_stride_scores,
                                       int64_t list_stride_idx, int n_lists, int64_t Q, int k_in, int k_out,
                                       float* out_scores, int64_t* out_idx, void* stream) {
  TFRS_CHECK_ARG(n_lists > 0 && Q >= 0 && k_in > 0 && k_out > 0 && k_out <= 2048, "topk_merge_strided: bad shape");
  TFRS_CHECK_ARG(list_stride_scores >= Q * k_in && list_stride_idx >= Q * k_in, "topk_merge_strided: list strides overlap");
  if (Q == 0) return TFRS_OK;
  TFRS_CHECK_ARG(scores && idx && out_scores && out_idx, "topk_merge_strided: NULL pointer");
  long long tot = (long long)n_lists * k_in;
  int ko = (int)(k_out < tot ? k_out : tot);
  MergeProvider prov{scores, (const long long*)idx, n_lists, Q, k_in, list_stride_scores, list_stride_idx};
  return launch_row_topk(prov, Q, ko, out_scores, (long long*)out_idx, k_out, (cudaStream_t)stream);
}

// ---- merge of SORTED lists (the sharded scan's all-gather) ---------------------------------------
// Every list is already in the total order (score desc, index asc), so two lists merge without a sort: the merged
// position of an element is (its position in its own list) + (how many elements of the partner list precede it),
// one binary search in shared memory.  Lists are merged pairwise in a tree (n -> n/2 -> ... -> 1), every level cut
// to k_out; the last level writes the result.  No atomics; ties between equal (score, index) pairs -- the
// (-inf, INT64_MAX) padding of short shards -- go to the lower list, so the order is total.
namespace tfrs {
constexpr int MS_THREADS = 256;
constexpr int MS_MAX_LISTS = 64;

__global__ void __launch_bounds__(MS_THREADS)
merge_sorted_kernel(const float* __restrict__ s, const long long* __restrict__ idx, long long stride_s, long long stride_i,
                    int n_lists, int k_in, int k_out, int region, float* __restrict__ out_s, long long* __restrict__ out_i,
                    int out_ld) {
  extern __shared__ __align__(16) unsigned char ms_smem[];
  // two ping-pong regions of `region` entries: indices (8 B) then scores (4 B)
  long long* ri[2] = {reinterpret_cast<long long*>(ms_smem), reinterpret_cast<long long*>(ms_smem) + region};
  float* rs[2] = {reinterpret_cast<float*>(ms_smem + (size_t)region * 16), reinterpret_cast<float*>(ms_smem + (size_t)region * 16) + region};
  __shared__ int lens[2][MS_MAX_LISTS];
  __shared__ float tau_sh;
  const long long row = blockIdx.x;
  const int total = n_lists * k_in;
  for (int t = threadIdx.x; t < total; t += MS_THREADS) {
    const int l = t / k_in, r = t - l * k_in;
    rs[0][t] = s[(long long)l * stride_s + row * k_in + r];
    ri[0][t] = idx[(long long)l * stride_i + row * k_in + r];
  }
  __syncthreads();
  // Pruning: with rr = ceil(k_out / n_lists), the first rr entries of every list are >= tau = min_l list_l[rr-1], so
  // at least k_out entries score >= tau and nothing scoring below tau can be in the result.
  const int rr = min(k_in, (k_out + n_lists - 1) / n_lists);
  if (threadIdx.x < 32) {
    float m = INFINITY;
    for (int l = threadIdx.x; l < n_lists; l += 32) m = fminf(m, rs[0][l * k_in + rr - 1]);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fminf(m, __shfl_xor_sync(0xffffffffu, m, o));
    if (threadIdx.x == 0) tau_sh = m;
  }
  __syncthreads();
  if (threadIdx.x < n_lists) {  // entries of this list that score >= tau (the list is descending)
    const float tau = tau_sh;
    const float* ls = rs[0] + threadIdx.x * k_in;
    int lo = rr, hi = k_in;
    while (lo < hi) { const int mid = (lo + hi) >> 1; if (ls[mid] >= tau) lo = mid + 1; else hi = mid; }
    lens[0][threadIdx.x] = lo;
  }
  __syncthreads();
  int n_prev = n_lists, c_prev = k_in, src = 0;
  for (;;) {
    const bool last = n_prev <= 2;
    const int c_new = min(k_out, 2 * c_prev);
    const float* ss = rs[src]; const long long* si = ri[src];
    float* ds = rs[src ^ 1]; long long* di = ri[src ^ 1];
    const int* ln = lens[src];
    int cap = 0;
    for (int l = 0; l < n_prev; ++l) cap = max(cap, ln[l]);
    const int slots = n_prev * cap;
    for (int t = threadIdx.x; t < slots; t += MS_THREADS) {
      const int l = t / cap, r = t - l * cap;
      if (r >= ln[l]) continue;
      const float es = ss[l * c_prev + r]; const long long ei = si[l * c_prev + r];
      const int m = l ^ 1;
      int rank = r;
      if (m < n_prev) {
        const float* ls = ss + m * c_prev; const long long* li = si + m * c_prev;
        int lo = 0, hi = ln[m];
        while (lo < hi) {  // first position of the partner list whose element does not precede e
          const int mid = (lo + hi) >> 1;
          const float xs = ls[mid];
          bool precedes = xs > es;
          if (xs == es) { const long long xi = li[mid]; precedes = (m < l) ? (xi <= ei) : (xi < ei); }
          if (precedes) lo = mid + 1; else hi = mid;
        }
        rank += lo;
      }
      if (rank < c_new) {
        if (last) { out_s[row * out_ld + rank] = es; out_i[row * out_ld + rank] = ei; }
        else { const int o = (l >> 1) * c_new + rank; ds[o] = es; di[o] = ei; }
      }
    }
    if (last) break;
    const int n_new = (n_prev + 1) >> 1;
    if (threadIdx.x < n_new) {
      const int a = ln[2 * threadIdx.x], b2 = (2 * threadIdx.x + 1 < n_prev) ? ln[2 * threadIdx.x + 1] : 0;
      lens[src ^ 1][threadIdx.x] = min(c_new, a + b2);
    }
    __syncthreads();
    n_prev = n_new; c_prev = c_new; src ^= 1;
  }
}
}  // namespace tfrs

extern "C" int tfrs_topk_merge_sorted_strided(const float* scores, const int64_t* idx, int64_t list_stride_scores,
                                              int64_t list_stride_idx, int n_lists, int64_t Q, int k_in, int k_out,
                                              float* out_scores, int64_t* out_idx, void* stream) {
  TFRS_CHECK_ARG(n_lists > 0 && Q >= 0 && k_in > 0 && k_out > 0, "topk_merge_sorted: bad shape");
  TFRS_CHECK_ARG(list_stride_scores >= Q * k_in && list_stride_idx >= Q * k_in, "topk_merge_sorted: list strides overlap");
  if (Q == 0) return TFRS_OK;
  TFRS_CHECK_ARG(scores && idx && out_scores && out_idx, "topk_merge_sorted: NULL pointer");
  const long long tot = (long long)n_lists * k_in;
  const int ko = (int)(k_out < tot ? k_out : tot);
  long long region = tot;  // largest level of the merge tree (entries)
  for (long long n = n_lists, c = k_in; n > 2;) { n = (n + 1) / 2; c = (2 * c < ko ? 2 * c : ko); if (n * c > region) region = n * c; }
  if (n_lists > MS_MAX_LISTS || region * 24 > 160 * 1024 || k_out > 2048)  // outside the tree merge: the sorting merge is always valid
    return tfrs_topk_merge_strided(scores, idx, list_stride_scores, list_stride_idx, n_lists, Q, k_in, k_out, out_scores, out_idx, stream);
  const size_t smem = (size_t)region * 24;
  TFRS_DYN_SMEM(merge_sorted_kernel, 160 * 1024);
  merge_sorted_kernel<<<(unsigned)Q, MS_THREADS, smem, (cudaStream_t)stream>>>(scores, (const long long*)idx, list_stride_scores,
                                                                             list_stride_idx, n_lists, k_in, ko, (int)region,
                                                                             out_scores, (long long*)out_idx, k_out);
  TFRS_LAUNCH_CHECK();
  return TFRS_OK;
}

// ---- exact score helpers ---------------------------------------------------------------------
namespace tfrs {
struct EpiStoreAcc {
  float* C; long long ldc; bool acc;
  __device__ __forceinline__ void operator()(int m, int n, float v, int) const {
    float* p = C + (long long)m * ldc + n;
    *p = acc ? (*p + v) : v;
  }
};
__global__ void __launch_bounds__(256)
rowwise_dot_kernel(const float* __restrict__ a, const float* __restrict__ b, long long rows, int d, float* __restrict__ out) {
  long long i = (long long)blockIdx.x * 256 + threadIdx.x;
  if (i >= rows) return;
  out[i] = dot_chain(a + i * d, b + i * d, d);
}
}  // namespace tfrs

extern "C" int tfrs_sgemm_f32(int transA, int transB, int64_t M, int64_t N, int64_t K, const float* A, int64_t lda,
                              const float* B, int64_t ldb, float* C, int64_t ldc, int accumulate, void* stream) {
  TFRS_CHECK_ARG(M >= 0 && N >= 0 && K >= 0 && M < (1ll << 31) && N < (1ll << 31) && K < (1ll << 31), "sgemm: bad shape");
  if (M == 0 || N == 0) return TFRS_OK;
  // K == 0: C = 0 (or C += 0); A and B are never read, and an empty operand may well be NULL
  TFRS_CHECK_ARG(C && (K == 0 || (A && B)), "sgemm: NULL pointer");
  cudaStream_t st = (cudaStream_t)stream;
  EpiStoreAcc epi{C, ldc, accumulate != 0};
  if (!transA && transB) return launch_sgemm<false, true>(A, lda, B, ldb, (int)M, (int)N, (int)K, 1, epi, st);
  if (!transA && !transB) return launch_sgemm<false, false>(A, lda, B, ldb, (int)M, (int)N, (int)K, 1, epi, st);
  if (transA && !transB) return launch_sgemm<true, false>(A, lda, B, ldb, (int)M, (int)N, (int)K, 1, epi, st);
  return launch_sgemm<true, true>(A, lda, B, ldb, (int)M, (int)N, (int)K, 1, epi, st);
}

extern "C" int tfrs_rowwise_dot_f32(const float* a, const float* b, int64_t rows, int d, float* out, void* stream) {
  TFRS_CHECK_ARG(rows >= 0 && d > 0, "rowwise_dot: bad shape");
  if (rows == 0) return TFRS_OK;
  TFRS_CHECK_ARG(a && b && out, "rowwise_dot: NULL pointer");
  rowwise_dot_kernel<<<(unsigned)ceil_div(rows, 256), 256, 0, (cudaStream_t)stream>>>(a, b, rows, d, out);
  TFRS_LAUNCH_CHECK();
  return TFRS_OK;
}
