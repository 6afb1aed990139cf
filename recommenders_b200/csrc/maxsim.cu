// maxsim.cu -- multi-interest ("multi-head") retrieval: a query is H vectors and scores a candidate by its best head,
// m(q, c) = max_h q_h . c (tasks/retrieval.py:172-176, the score the maxsim loss trains).
//   tfrs_topk_maxsim_merge_f32 (K26) : H per-head top-w lists of a query -> its maxsim top-k_out (DESIGN.md, K26)
//   tfrs_rowwise_maxsim_f32          : max_h dot(q[r, h], c[r]), FactorizedTopK's positive score for [R, H, d] queries
// Deterministic: integer atomics only, and their outcome does not depend on their order.
#include "common.cuh"

namespace tfrs {

constexpr int MM_THREADS = 256;

// entry t of a query's H*w entries (t = h * w + r): (order key of the score, inverted position) -- the larger key is the
// higher score, then the lower head.  Never 0 (the low half is nonzero for t < 2^32 - 1), so 0 marks an empty slot.
__device__ __forceinline__ unsigned long long mm_key(float s, int t) {
  return ((unsigned long long)okey(s + 0.0f) << 32) | (unsigned long long)(0xFFFFFFFFu - (unsigned int)t);
}

__device__ __forceinline__ int mm_pos(unsigned long long key) { return (int)(0xFFFFFFFFu - (unsigned int)key); }

__device__ __forceinline__ unsigned int mm_slot(long long i, unsigned int T) {
  unsigned long long x = (unsigned long long)i;   // fmix64 of MurmurHash3, then the high word scaled onto [0, T)
  x ^= x >> 33; x *= 0xff51afd7ed558ccdull; x ^= x >> 33; x *= 0xc4ceb9fe1a85ec53ull; x ^= x >> 33;
  return (unsigned int)(((x >> 32) * (unsigned long long)T) >> 32);
}

// the hash slot of candidate `id` (present in the table)
__device__ __forceinline__ unsigned int mm_find(const unsigned long long* tab, const long long* mi, long long id,
                                                unsigned int T) {
  unsigned int slot = mm_slot(id, T);
  while (mi[mm_pos(tab[slot])] != id) slot = (slot + 1 == T) ? 0 : slot + 1;
  return slot;
}

// Table slots for n entries: load factor <= 2/3 with linear probing, and always one empty slot.
static inline unsigned int mm_table_slots(int n) { return (unsigned int)(n + n / 2 + 1); }

static inline size_t mm_smem_bytes(int H, int w) {
  const int n = H * w;
  return (size_t)n * 8 + (size_t)mm_table_slots(n) * 8 + (size_t)n * 4 + (size_t)H * (w + 1) * 2;
}

// One CTA per query.  Shared memory: the entries' indices and scores, the hash table keyed by candidate index, and per
// list the prefix counts of its surviving entries (uint16: w <= TFRS_MAXSIM_MAX_ENTRIES).
__global__ void __launch_bounds__(MM_THREADS)
maxsim_merge_kernel(const float* __restrict__ scores, const long long* __restrict__ idx, int H, int w, int k_out,
                    unsigned int T, float* __restrict__ out_s, long long* __restrict__ out_i) {
  extern __shared__ __align__(16) unsigned char mm_smem[];
  const int n = H * w;
  long long* mi = reinterpret_cast<long long*>(mm_smem);
  unsigned long long* tab = reinterpret_cast<unsigned long long*>(mm_smem + (size_t)n * 8);
  float* ms = reinterpret_cast<float*>(mm_smem + (size_t)n * 8 + (size_t)T * 8);
  unsigned short* pre = reinterpret_cast<unsigned short*>(mm_smem + (size_t)n * 12 + (size_t)T * 8);   // [H][w + 1]
  const long long row = blockIdx.x;
  for (int t = threadIdx.x; t < n; t += MM_THREADS) { ms[t] = scores[row * n + t]; mi[t] = idx[row * n + t]; }
  for (unsigned int t = threadIdx.x; t < T; t += MM_THREADS) tab[t] = 0ull;
  __syncthreads();

  // 1. one entry per candidate index: the slot of an index ends at the maximum key of its entries
  for (int t = threadIdx.x; t < n; t += MM_THREADS) {
    const unsigned long long mine = mm_key(ms[t], t);
    const long long id = mi[t];
    unsigned int slot = mm_slot(id, T);
    for (;;) {
      const unsigned long long old = atomicCAS(&tab[slot], 0ull, mine);
      if (old == 0ull) break;
      if (mi[mm_pos(old)] == id) { atomicMax(&tab[slot], mine); break; }   // a slot never changes its index
      slot = (slot + 1 == T) ? 0 : slot + 1;
    }
  }
  __syncthreads();

  // 2. a warp per list: pre[l][r] = #{surviving entries among the first r of list l}
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int l = warp; l < H; l += MM_THREADS / 32) {
    unsigned short* pl = pre + (size_t)l * (w + 1);
    int base = 0;
    if (lane == 0) pl[0] = 0;
    for (int r0 = 0; r0 < w; r0 += 32) {
      const int r = r0 + lane, t = l * w + r;
      const bool keep = r < w && tab[mm_find(tab, mi, mi[t], T)] == mm_key(ms[t], t);
      const unsigned int b = __ballot_sync(0xffffffffu, keep);
      if (r < w) pl[r + 1] = (unsigned short)(base + __popc(b & (0xffffffffu >> (31 - lane))));
      base += __popc(b);
    }
  }
  __syncthreads();

  // 3. the merged rank of a surviving entry: survivors ahead of it in its own list, plus in every other list the
  //    survivors among the entries that precede it (one binary search; every list is sorted in that order)
  for (int t = threadIdx.x; t < n; t += MM_THREADS) {
    const int l = t / w, r = t - l * w;
    const unsigned short* pl = pre + (size_t)l * (w + 1);
    if (pl[r + 1] == pl[r]) continue;
    const float es = ms[t];
    const long long ei = mi[t];
    int rank = pl[r];
    for (int m = 0; m < H && rank < k_out; ++m) {
      if (m == l) continue;
      const float* ls = ms + (size_t)m * w;
      const long long* li = mi + (size_t)m * w;
      int lo = 0, hi = w;
      while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (better(ls[mid], li[mid], es, ei)) lo = mid + 1; else hi = mid;
      }
      rank += pre[(size_t)m * (w + 1) + lo];
    }
    if (rank < k_out) { out_s[row * k_out + rank] = es; out_i[row * k_out + rank] = ei; }
  }
}

__global__ void __launch_bounds__(256)
rowwise_maxsim_kernel(const float* __restrict__ q, const float* __restrict__ c, long long rows, int H, int d,
                      float* __restrict__ out) {
  const long long i = (long long)blockIdx.x * 256 + threadIdx.x;
  if (i >= rows) return;
  const float* pc = c + i * d;
  const float* pq = q + i * H * d;
  float best = dot_chain(pq, pc, d);
  for (int h = 1; h < H; ++h) {
    const float s = dot_chain(pq + (long long)h * d, pc, d);
    if (s > best) best = s;   // ties (+-0 included) keep the lower head's bits
  }
  out[i] = best;
}

}  // namespace tfrs
using namespace tfrs;

extern "C" int tfrs_topk_maxsim_merge_f32(const float* scores, const int64_t* idx, int64_t Q, int H, int w, int k_out,
                                          float* out_scores, int64_t* out_idx, void* stream) {
  TFRS_CHECK_ARG(Q >= 0 && Q < (1ll << 31) && H > 0 && w > 0 && k_out > 0 && k_out <= w,
                 "maxsim_merge: bad shape (Q=%lld H=%d w=%d k_out=%d; needs 1 <= k_out <= w)", (long long)Q, H, w, k_out);
  if ((long long)H * w > TFRS_MAXSIM_MAX_ENTRIES) {
    set_error("maxsim_merge: H=%d heads of w=%d entries is %lld entries per query, above %d", H, w, (long long)H * w,
              TFRS_MAXSIM_MAX_ENTRIES);
    return TFRS_ERR_UNSUPPORTED;
  }
  if (Q == 0) return TFRS_OK;
  TFRS_CHECK_ARG(scores && idx && out_scores && out_idx, "maxsim_merge: NULL pointer");
  const size_t smem = mm_smem_bytes(H, w);
  TFRS_DYN_SMEM(maxsim_merge_kernel, mm_smem_bytes(TFRS_MAXSIM_MAX_ENTRIES, 1));   // the largest layout: w = 1
  maxsim_merge_kernel<<<(unsigned)Q, MM_THREADS, smem, (cudaStream_t)stream>>>(
      scores, (const long long*)idx, H, w, k_out, mm_table_slots(H * w), out_scores, (long long*)out_idx);
  TFRS_LAUNCH_CHECK();
  return TFRS_OK;
}

extern "C" int tfrs_rowwise_maxsim_f32(const float* q, const float* c, int64_t rows, int H, int d, float* out,
                                       void* stream) {
  TFRS_CHECK_ARG(rows >= 0 && H > 0 && d > 0, "rowwise_maxsim: bad shape (rows=%lld H=%d d=%d)", (long long)rows, H, d);
  if (rows == 0) return TFRS_OK;
  TFRS_CHECK_ARG(q && c && out, "rowwise_maxsim: NULL pointer");
  rowwise_maxsim_kernel<<<(unsigned)ceil_div(rows, 256), 256, 0, (cudaStream_t)stream>>>(q, c, rows, H, d, out);
  TFRS_LAUNCH_CHECK();
  return TFRS_OK;
}
