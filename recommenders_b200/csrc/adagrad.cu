// adagrad.cu -- K4: deterministic sparse Adagrad on the rows touched by a batch.
// Replaces optimizer.apply_gradients(IndexedSlices) (models/base.py:77-78, Adagrad per README.md:84).
//   1. keys = (id << 24 | position) grouped by id with positions ascending: bucketed rank sort for a training-step batch
//      (n <= 16384), bitonic sort (shared-memory tiles + global strides) beyond
//   2. one warp per run of equal ids: duplicate gradient rows are summed in order of occurrence
//      (lanes = columns, no float atomics), then  acc += g*g ; var -= lr*g/sqrt(acc+eps)  (or the
//      legacy sqrt(acc)+eps form).  Every step is a single IEEE fp32 op (no FMA contraction) so the
//      result is bit-identical to oracle/tfrs_oracle.c::orc_sparse_adagrad.
// HBM-bound: algorithmic bytes = unique_rows * d * 4 * 4 (table r/w + accum r/w) + n*d*4 (grads).
#include "adagrad.cuh"

namespace tfrs {

constexpr int AG_TILE = 8192;       // keys per CTA tile (64 KB of shared memory)
constexpr int AG_THREADS = 1024;
constexpr unsigned long long AG_INVALID = ~0ull;

template <typename IdT>
__device__ __forceinline__ unsigned long long ag_key(const IdT* __restrict__ ids, long long j, long long rows) {
  const long long r = (long long)ids[j];
  return (((r >= 0 && r < rows) ? (unsigned long long)r : AG_BAD_ID) << 24) | (unsigned long long)j;
}


template <typename IdT>
__global__ void ag_build_keys(const IdT* __restrict__ ids, long long n, long long rows, long long P,
                              unsigned long long* __restrict__ keys) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= P) return;
  keys[i] = i < n ? ag_key(ids, i, rows) : AG_INVALID;   // padding (~0) and out-of-range ids (AG_BAD_ID) sort last
}

__device__ __forceinline__ void ag_cmpswap(unsigned long long& a, unsigned long long& b, bool asc) {
  if ((a > b) == asc) { unsigned long long t = a; a = b; b = t; }
}

// Sorts (first_size == 2) or merges (first_size == size) one AG_TILE chunk in shared memory.
// Processes bitonic stages size = first_size..last_size with strides min(size/2, TILE/2)..1.
__global__ void __launch_bounds__(AG_THREADS)
ag_bitonic_local(unsigned long long* __restrict__ keys, long long P, long long first_size, long long last_size) {
  extern __shared__ unsigned long long sk[];
  const long long base = (long long)blockIdx.x * AG_TILE;
  const int tile = (int)min((long long)AG_TILE, P - base);
  for (int t = threadIdx.x; t < tile; t += AG_THREADS) sk[t] = keys[base + t];
  __syncthreads();
  for (long long size = first_size; size <= last_size; size <<= 1) {
    int s0 = (int)min(size >> 1, (long long)(tile >> 1));
    for (int stride = s0; stride > 0; stride >>= 1) {
      for (int t = threadIdx.x; t < (tile >> 1); t += AG_THREADS) {
        int lo = 2 * t - (t & (stride - 1));
        int hi = lo + stride;
        bool asc = (((base + lo) & size) == 0);
        unsigned long long a = sk[lo], b = sk[hi];
        ag_cmpswap(a, b, asc);
        sk[lo] = a; sk[hi] = b;
      }
      __syncthreads();
    }
  }
  for (int t = threadIdx.x; t < tile; t += AG_THREADS) keys[base + t] = sk[t];
}

// n <= AG_RANK_MAX: bucketed RANK sort.  ag_apply only needs the members of an id to be contiguous and in order of
// occurrence -- not a global order by id.  So: (1) one CTA hashes the ids into AB_BUCKETS buckets (shared-memory histogram,
// exclusive scan, scatter: equal ids land in the same bucket); (2) keys are unique (the position is part of the key), so the
// slot of a key inside its bucket is the number of bucket members below it: every thread owns one key and counts over its
// bucket only (n^2 / AB_BUCKETS comparisons instead of n^2; the all-pairs count over the whole batch was 56 us of the 80 us
// step at cfg3).  The result is deterministic: the scatter order inside a bucket is not, the ranks are.
constexpr int AG_RANK_MAX = 16384;
constexpr int AB_BUCKETS = 256, AB_THREADS = 1024, AB_PER_THREAD = AG_RANK_MAX / AB_THREADS, AB_SPLIT = 8;
__device__ __forceinline__ int ag_bucket(unsigned long long key) {
  const unsigned int id = (unsigned int)(key >> 24) ^ (unsigned int)(key >> 56);
  return (int)((id * 0x9E3779B1u) >> 24);   // 8 bits
}
// one CTA: the batch's keys live in registers between the histogram and the scatter pass
template <typename IdT>
__global__ void __launch_bounds__(AB_THREADS)
ag_bucket_scatter(const IdT* __restrict__ ids, long long n, long long rows, unsigned long long* __restrict__ bkeys,
                  unsigned int* __restrict__ bstart, unsigned int* __restrict__ rank) {
  __shared__ unsigned int hist[AB_BUCKETS], cur[AB_BUCKETS];
  unsigned long long k[AB_PER_THREAD];
#pragma unroll
  for (int u = 0; u < AB_PER_THREAD; ++u) {
    const long long j = threadIdx.x + (long long)u * AB_THREADS;
    k[u] = j < n ? ag_key(ids, j, rows) : ~0ull;
    if (j < n) rank[j] = 0;
  }
  if (threadIdx.x < AB_BUCKETS) hist[threadIdx.x] = 0;
  __syncthreads();
#pragma unroll
  for (int u = 0; u < AB_PER_THREAD; ++u)
    if (k[u] != ~0ull) atomicAdd(&hist[ag_bucket(k[u])], 1u);
  __syncthreads();
  if (threadIdx.x < 32) {   // exclusive scan of the 256 counters: 8 per lane + a warp scan
    unsigned int c[8], tot = 0;
#pragma unroll
    for (int i = 0; i < 8; ++i) { c[i] = hist[threadIdx.x * 8 + i]; tot += c[i]; }
    unsigned int inc = tot;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const unsigned int v = __shfl_up_sync(0xffffffffu, inc, o); if ((int)threadIdx.x >= o) inc += v; }
    unsigned int a = inc - tot;
#pragma unroll
    for (int i = 0; i < 8; ++i) { cur[threadIdx.x * 8 + i] = a; bstart[threadIdx.x * 8 + i] = a; a += c[i]; }
    if (threadIdx.x == 31) bstart[AB_BUCKETS] = a;
  }
  __syncthreads();
#pragma unroll
  for (int u = 0; u < AB_PER_THREAD; ++u)
    if (k[u] != ~0ull) bkeys[atomicAdd(&cur[ag_bucket(k[u])], 1u)] = k[u];
}
// rank of a key inside its bucket = number of bucket members below it; blockIdx.y takes one slice of the bucket, so a hot
// id's bucket (a tenth of a Zipf batch) is counted by AB_SPLIT threads per key instead of one
__global__ void __launch_bounds__(128)
ag_bucket_rank(const unsigned long long* __restrict__ bkeys, long long n, const unsigned int* __restrict__ bstart,
               unsigned int* __restrict__ rank) {
  const long long i = (long long)blockIdx.x * 128 + threadIdx.x;
  if (i >= n) return;
  const unsigned long long mine = bkeys[i];
  const int b = ag_bucket(mine);
  const unsigned int s = bstart[b], e = bstart[b + 1];
  const unsigned int per = (e - s + AB_SPLIT - 1) / AB_SPLIT;
  unsigned int j = s + blockIdx.y * per;
  const unsigned int j1 = min(e, j + per);
  unsigned int r = 0;
  for (; j + 8 <= j1; j += 8) {   // lanes of a warp mostly share the bucket: broadcast loads, 8 in flight
    unsigned long long kk[8];
#pragma unroll
    for (int u = 0; u < 8; ++u) kk[u] = __ldg(bkeys + j + u);
#pragma unroll
    for (int u = 0; u < 8; ++u) r += kk[u] < mine;
  }
  for (; j < j1; ++j) r += __ldg(bkeys + j) < mine;
  if (r) atomicAdd(&rank[i], r);
}
__global__ void __launch_bounds__(256)
ag_bucket_place(const unsigned long long* __restrict__ bkeys, long long n, const unsigned int* __restrict__ bstart,
                const unsigned int* __restrict__ rank, unsigned long long* __restrict__ keys) {
  const long long i = (long long)blockIdx.x * 256 + threadIdx.x;
  if (i >= n) return;
  const unsigned long long mine = bkeys[i];
  keys[bstart[ag_bucket(mine)] + rank[i]] = mine;
}

__global__ void ag_bitonic_global(unsigned long long* __restrict__ keys, long long P, long long size, long long stride) {
  long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= (P >> 1)) return;
  long long lo = 2 * t - (t & (stride - 1));
  long long hi = lo + stride;
  bool asc = ((lo & size) == 0);
  unsigned long long a = keys[lo], b = keys[hi];
  ag_cmpswap(a, b, asc);
  keys[lo] = a; keys[hi] = b;
}

// One warp per run of equal ids (the warp of the run's first slot; the others exit).  Duplicates are summed in order of
// occurrence -- the keys are sorted by (id, position) -- with the gradient rows of 8 members in flight per step, so a hot
// id's chain costs one DRAM round trip per 8 members instead of two per member.  Runs longer than AG_LONG members are left
// to ag_apply_long (a whole CTA stages their rows through shared memory).
__device__ __forceinline__ void ag_update(float* __restrict__ trow, float* __restrict__ arow, int c, float g, float lr, float eps, int eps_inside) {
  const float a = __fadd_rn(arow[c], __fmul_rn(g, g));
  arow[c] = a;
  const float den = eps_inside ? __fsqrt_rn(__fadd_rn(a, eps)) : __fadd_rn(__fsqrt_rn(a), eps);
  trow[c] = __fsub_rn(trow[c], __fdiv_rn(__fmul_rn(lr, g), den));
}

__global__ void __launch_bounds__(256)
ag_apply(const unsigned long long* __restrict__ keys, long long n, const float* __restrict__ grad, int d,
         float* __restrict__ table, float* __restrict__ accum, float lr, float eps, int eps_inside,
         unsigned int* __restrict__ long_count, unsigned int* __restrict__ long_list) {
  const long long i = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;  // one warp per sorted slot
  const int lane = threadIdx.x & 31;
  unsigned long long id;
  if (i >= n || !ag_run_head(keys, i, id)) return;
  // run length: ballots over 32-slot windows
  long long end = i + 1;
  for (;;) {
    const long long j = end + lane;
    const bool same = j < n && (keys[j] >> 24) == id;
    const unsigned int vote = __ballot_sync(0xffffffffu, same);
    const int run = __ffs(~vote) - 1;          // leading members of this window (32 when all match: ~vote == 0 -> ffs 0 -> -1)
    if (vote == 0xffffffffu) { end += 32; if (end - i > AG_LONG) break; continue; }
    end += run;
    break;
  }
  if (end - i > AG_LONG) {   // hot id: hand the run to the CTA-wide kernel
    if (lane == 0) long_list[atomicAdd(long_count, 1u)] = (unsigned int)i;
    return;
  }
  float* trow = table + (long long)id * d;
  float* arow = accum + (long long)id * d;
  const int L = (int)(end - i);
  for (int c = lane; c < d; c += 32) {
    float g = 0.f;
    for (int m0 = 0; m0 < L; m0 += 8) {
      float v[8];
#pragma unroll
      for (int u = 0; u < 8; ++u)
        v[u] = (m0 + u < L) ? __ldg(grad + (long long)(keys[i + m0 + u] & 0xFFFFFFull) * d + c) : 0.f;
#pragma unroll
      for (int u = 0; u < 8; ++u)
        if (m0 + u < L) g = (m0 + u == 0) ? v[u] : __fadd_rn(g, v[u]);
    }
    ag_update(trow, arow, c, g, lr, eps, eps_inside);
  }
}

// Hot ids (Zipf batches: one id can own a tenth of the batch): one CTA per long run.  All 256 threads stream the run's
// gradient rows into a shared-memory tile (AL_ROWS rows in flight per step), then one thread per column adds the tile's
// rows IN ORDER -- the chain is fp32 adds on shared memory, not DRAM round trips.
__global__ void __launch_bounds__(AL_THREADS)
ag_apply_long(const unsigned long long* __restrict__ keys, long long n, const float* __restrict__ grad, int d,
              float* __restrict__ table, float* __restrict__ accum, float lr, float eps, int eps_inside,
              const unsigned int* __restrict__ long_count, const unsigned int* __restrict__ long_list, int tile_rows) {
  extern __shared__ __align__(16) float al_tile[];   // [tile_rows][d]
  __shared__ unsigned int pos_sh[AL_ROWS];
  for (unsigned int w = blockIdx.x; w < *long_count; w += gridDim.x) {
    const long long i = long_list[w];
    const unsigned long long id = keys[i] >> 24;
    // run end: 256 sorted keys per step (the members form a contiguous prefix of every window)
    long long end = i + 1;
    for (;;) {
      const long long j = end + threadIdx.x;
      const int same = (j < n && (keys[j] >> 24) == id) ? 1 : 0;
      const int cnt = __syncthreads_count(same);
      end += cnt;
      if (cnt < AL_THREADS) break;
    }
    float acc_g[4];   // a thread owns columns threadIdx.x + 256*u (d <= 1024)
#pragma unroll
    for (int u = 0; u < 4; ++u) acc_g[u] = 0.f;
    for (long long m0 = i; m0 < end; m0 += tile_rows) {
      const int rows_here = (int)min((long long)tile_rows, end - m0);
      // the tile's gradient-row numbers first (one coalesced read), then every thread has 4 independent 16-byte row
      // loads in flight: one DRAM round trip per tile instead of one per element.  float4 only when every row starts on
      // a 16-byte boundary: a contiguous view may start 4, 8 or 12 bytes into its storage
      if ((int)threadIdx.x < rows_here) pos_sh[threadIdx.x] = (unsigned int)(keys[m0 + threadIdx.x] & 0xFFFFFFull);
      __syncthreads();
      if ((d & 3) == 0 && (reinterpret_cast<uintptr_t>(grad) & 15) == 0) {
        const unsigned int d4 = (unsigned int)d >> 2, total4 = (unsigned int)rows_here * d4;
        for (unsigned int e0 = threadIdx.x; e0 < total4; e0 += AL_THREADS * 4) {
          float4 v[4];
#pragma unroll
          for (int u = 0; u < 4; ++u) {
            const unsigned int e = e0 + u * AL_THREADS;
            if (e < total4) { const unsigned int r = e / d4, c4 = e - r * d4; v[u] = __ldg(reinterpret_cast<const float4*>(grad + (long long)pos_sh[r] * d) + c4); }
          }
#pragma unroll
          for (int u = 0; u < 4; ++u) {
            const unsigned int e = e0 + u * AL_THREADS;
            if (e < total4) reinterpret_cast<float4*>(al_tile)[e] = v[u];
          }
        }
      } else {
        for (int e = threadIdx.x; e < rows_here * d; e += AL_THREADS) {
          const int r = e / d, c = e - r * d;
          al_tile[e] = __ldg(grad + (long long)pos_sh[r] * d + c);
        }
      }
      __syncthreads();
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int c = threadIdx.x + AL_THREADS * u;
        if (c < d) {
          float g = acc_g[u];
          for (int r = 0; r < rows_here; ++r) g = (m0 == i && r == 0) ? al_tile[c] : __fadd_rn(g, al_tile[r * d + c]);
          acc_g[u] = g;
        }
      }
      __syncthreads();
    }
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int c = threadIdx.x + AL_THREADS * u;
      if (c < d) ag_update(table + (long long)id * d, accum + (long long)id * d, c, acc_g[u], lr, eps, eps_inside);
    }
    __syncthreads();
  }
}

static long long ag_pow2(long long n) { long long p = 1; while (p < n) p <<= 1; return p; }

int ag_check_args(const char* who, bool state, long long rows, int d, int ids_dtype, long long n, const void* ids,
                  const void* grad) {
  TFRS_CHECK_ARG(state && rows > 0 && d > 0, "%s: bad table", who);
  TFRS_CHECK_ARG(ids_dtype == TFRS_I32 || ids_dtype == TFRS_I64, "%s: ids_dtype must be I32 or I64", who);
  TFRS_CHECK_ARG(n >= 0 && n < (1ll << 24), "%s: n=%lld must be < 2^24", who, n);
  TFRS_CHECK_ARG(rows < (1ll << 40), "%s: rows must be < 2^40", who);
  TFRS_CHECK_ARG(n == 0 || (ids && grad), "%s: NULL ids/grad", who);
  return TFRS_OK;
}

size_t ag_group_workspace_bytes(long long n) {
  const size_t P = (size_t)ag_pow2(n > 2 ? n : 2);
  return P * 8 /*keys*/ + P * 8 /*bucketed keys*/ + P * 4 /*ranks*/ + (P / AG_LONG + 2) * 4 /*long-run list*/ + (AB_BUCKETS + 1) * 4 + 1024;
}

int ag_group(const void* ids, int ids_dtype, long long n, long long rows, void* ws, cudaStream_t st, AgGroups* out) {
  const long long P = ag_pow2(n > 2 ? n : 2);
  unsigned long long* keys = (unsigned long long*)ws;
  unsigned long long* bkeys = keys + P;
  unsigned int* long_count = (unsigned int*)(bkeys + P);
  unsigned int* long_list = long_count + 1;
  unsigned int* bstart = long_list + (P / AG_LONG + 1);
  unsigned int* rank = bstart + AB_BUCKETS + 1;
  *out = AgGroups{keys, long_count, long_list};
  if (n <= AG_RANK_MAX) {
    if (ids_dtype == TFRS_I32) ag_bucket_scatter<int32_t><<<1, AB_THREADS, 0, st>>>((const int32_t*)ids, n, rows, bkeys, bstart, rank);
    else ag_bucket_scatter<int64_t><<<1, AB_THREADS, 0, st>>>((const int64_t*)ids, n, rows, bkeys, bstart, rank);
    TFRS_LAUNCH_CHECK();
    ag_bucket_rank<<<dim3((unsigned)ceil_div(n, 128), AB_SPLIT), 128, 0, st>>>(bkeys, n, bstart, rank);
    TFRS_LAUNCH_CHECK();
    ag_bucket_place<<<(unsigned)ceil_div(n, 256), 256, 0, st>>>(bkeys, n, bstart, rank, keys);
    TFRS_LAUNCH_CHECK();
    return TFRS_OK;
  }
  return ag_sort(ids, ids_dtype, n, rows, ws, st);
}

int ag_sort(const void* ids, int ids_dtype, long long n, long long rows, void* ws, cudaStream_t st) {
  const long long P = ag_pow2(n > 2 ? n : 2);
  unsigned long long* keys = (unsigned long long*)ws;
  unsigned kb = (unsigned)ceil_div(P, 256);
  if (ids_dtype == TFRS_I32) ag_build_keys<int32_t><<<kb, 256, 0, st>>>((const int32_t*)ids, n, rows, P, keys);
  else ag_build_keys<int64_t><<<kb, 256, 0, st>>>((const int64_t*)ids, n, rows, P, keys);
  TFRS_LAUNCH_CHECK();
  TFRS_DYN_SMEM(ag_bitonic_local, AG_TILE * 8);
  const unsigned tiles = (unsigned)ceil_div(P, AG_TILE);
  const long long local_max = P < AG_TILE ? P : AG_TILE;
  ag_bitonic_local<<<tiles, AG_THREADS, AG_TILE * 8, st>>>(keys, P, 2, local_max);
  TFRS_LAUNCH_CHECK();
  for (long long size = 2ll * AG_TILE; size <= P; size <<= 1) {
    for (long long stride = size >> 1; stride >= AG_TILE; stride >>= 1) {
      ag_bitonic_global<<<(unsigned)ceil_div(P >> 1, 256), 256, 0, st>>>(keys, P, size, stride);
      TFRS_LAUNCH_CHECK();
    }
    ag_bitonic_local<<<tiles, AG_THREADS, AG_TILE * 8, st>>>(keys, P, size, size);
    TFRS_LAUNCH_CHECK();
  }
  return TFRS_OK;
}

}  // namespace tfrs
using namespace tfrs;

extern "C" size_t tfrs_sparse_adagrad_workspace_bytes(int64_t n, int d) {
  (void)d;
  return ag_group_workspace_bytes(n);
}

extern "C" int tfrs_sparse_adagrad_f32(float* table, float* accum, int64_t rows, int d, const void* ids,
                                       int ids_dtype, int64_t n, const float* grad_rows, float lr, float eps,
                                       int eps_inside_sqrt, void* ws, size_t ws_bytes, void* stream) {
  int rc;
  if ((rc = ag_check_args("sparse_adagrad", table && accum, rows, d, ids_dtype, n, ids, grad_rows)) != TFRS_OK) return rc;
  if (n == 0) return TFRS_OK;
  TFRS_CHECK_ARG(d <= 1024, "sparse_adagrad: d=%d > 1024", d);
  if (!ws || ws_bytes < tfrs_sparse_adagrad_workspace_bytes(n, d)) { set_error("sparse_adagrad: workspace too small"); return TFRS_ERR_WORKSPACE_TOO_SMALL; }
  cudaStream_t st = (cudaStream_t)stream;
  AgGroups gr;
  if ((rc = ag_group(ids, ids_dtype, n, rows, ws, st, &gr)) != TFRS_OK) return rc;
  TFRS_CUDA(cudaMemsetAsync(gr.long_count, 0, 4, st));
  ag_apply<<<(unsigned)ceil_div(n * 32, 256), 256, 0, st>>>(gr.keys, n, grad_rows, d, table, accum, lr, eps, eps_inside_sqrt,
                                                            gr.long_count, gr.long_list);
  TFRS_LAUNCH_CHECK();
  int tile_rows = (64 * 1024) / (d * 4); if (tile_rows > AL_ROWS) tile_rows = AL_ROWS; if (tile_rows < 1) tile_rows = 1;
  TFRS_DYN_SMEM(ag_apply_long, 64 * 1024);
  ag_apply_long<<<(unsigned)sm_count(), AL_THREADS, (size_t)tile_rows * d * 4, st>>>(gr.keys, n, grad_rows, d, table, accum, lr, eps,
                                                                                     eps_inside_sqrt, gr.long_count, gr.long_list, tile_rows);
  TFRS_LAUNCH_CHECK();
  return TFRS_OK;
}
