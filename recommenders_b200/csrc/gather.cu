// gather.cu -- K1: multi-table embedding row gather into a concatenated activation.
// Replaces tf.keras.layers.Embedding -> tf.gather (README.md:62-66,77-78).  HBM-bound:
// algorithmic bytes = n * sum(dims) * 4 read + the same written (+ ids).  One 16-byte lane per
// thread, consecutive threads cover one row (coalesced 128..256 B row reads and writes), the
// table is selected by blockIdx.y so the inner index math is a single divide.
#include "common.cuh"

namespace tfrs {

constexpr int GT_MAX_TABLES = 32;
constexpr int GT_THREADS = 256;
constexpr int GT_ROWS_PER_THREAD = 4;  // independent loads in flight per thread

struct GatherParams {
  const float* table[GT_MAX_TABLES];
  const void* ids[GT_MAX_TABLES];
  long long rows[GT_MAX_TABLES];
  int dim[GT_MAX_TABLES];
  int col_off[GT_MAX_TABLES];
};

template <typename IdT, bool VEC>
__global__ void __launch_bounds__(GT_THREADS)
gather_kernel(GatherParams p, long long n, float* __restrict__ out, long long out_ld) {
  const int t = blockIdx.y;
  const float* __restrict__ table = p.table[t];
  const IdT* __restrict__ ids = reinterpret_cast<const IdT*>(p.ids[t]);
  const long long rows = p.rows[t];
  const int dim = p.dim[t];
  const int lanes = VEC ? dim / 4 : dim;  // work items per row
  const int lane_shift = (lanes & (lanes - 1)) == 0 ? (31 - __clz(lanes)) : -1;
  const long long total = n * lanes;
  const long long stride = (long long)gridDim.x * GT_THREADS;
  long long w = (long long)blockIdx.x * GT_THREADS + threadIdx.x;
  // each thread handles GT_ROWS_PER_THREAD items `stride` apart: loads first, then stores
  for (; w < total; w += stride * GT_ROWS_PER_THREAD) {
    float4 v4[GT_ROWS_PER_THREAD]; float v1[GT_ROWS_PER_THREAD];
    long long dst[GT_ROWS_PER_THREAD];
#pragma unroll
    for (int u = 0; u < GT_ROWS_PER_THREAD; ++u) {
      long long e = w + u * stride;
      dst[u] = -1;
      if (e < total) {
        long long i; int l;
        if (lane_shift >= 0) { i = e >> lane_shift; l = (int)(e & (lanes - 1)); }   // lanes is a power of two: no division
        else if (total < (1ll << 32)) { unsigned int e32 = (unsigned int)e; i = e32 / (unsigned int)lanes; l = (int)(e32 - (unsigned int)i * lanes); }
        else { i = e / lanes; l = (int)(e - i * lanes); }
        long long r = (long long)ids[i];
        bool ok = (r >= 0 && r < rows);
        if (VEC) {
          v4[u] = ok ? __ldg(reinterpret_cast<const float4*>(table + r * dim) + l) : make_float4(0.f, 0.f, 0.f, 0.f);
          dst[u] = i * out_ld + p.col_off[t] + l * 4;
        } else {
          v1[u] = ok ? __ldg(table + r * dim + l) : 0.f;
          dst[u] = i * out_ld + p.col_off[t] + l;
        }
      }
    }
#pragma unroll
    for (int u = 0; u < GT_ROWS_PER_THREAD; ++u) {
      if (dst[u] >= 0) {
        if (VEC) *reinterpret_cast<float4*>(out + dst[u]) = v4[u];
        else out[dst[u]] = v1[u];
      }
    }
  }
}

// Variant "warp-chunk": a warp owns 32 consecutive batch rows of one table.  Lane l loads ids[i0+l] ONCE (one coalesced
// 128-byte read per 32 rows instead of a redundant id read per 16-byte lane), row ids travel by shuffle, and the
// warp then issues up to 8 independent 16-byte row reads per thread before the first store.
//
// Hot rows (skewed id distributions): a CTA covers GT_CTA_ROWS batch rows of one table.  Vocabularies are normally
// frequency-sorted, so the hot rows are the FIRST rows of the table: when more of the CTA's ids fall into the first H rows
// (H = GT_HOT_BYTES / row bytes) than the H rows it costs to fetch them, thread 0 stages that contiguous block in shared
// memory with one bulk-TMA copy (cp.async.bulk + mbarrier) and every hit is served from there -- duplicates of a hot row
// inside the chunk cost one L2 read instead of one each.  Uniform ids never trigger it (one block-wide count, no copy).
constexpr int GT_HOT_BYTES = 16384;
constexpr int GT_CTA_CHUNKS = 2;                          // 32-row chunks per warp
constexpr int GT_CTA_ROWS = (GT_THREADS / 32) * 32 * GT_CTA_CHUNKS;

template <typename IdT>
__global__ void __launch_bounds__(GT_THREADS)
gather_warpchunk_kernel(GatherParams p, long long n, float* __restrict__ out, long long out_ld) {
  __shared__ __align__(128) float4 hot[GT_HOT_BYTES / 16];
  __shared__ __align__(8) uint64_t hot_bar;
  const int t = blockIdx.y;
  const float4* __restrict__ table = reinterpret_cast<const float4*>(p.table[t]);
  const IdT* __restrict__ ids = reinterpret_cast<const IdT*>(p.ids[t]);
  const long long rows = p.rows[t];
  const int L = p.dim[t] >> 2;             // 16-byte lanes per row: power of two, <= 32 (checked by the host)
  const int lshift = 31 - __clz(L);
  const int R = 32 >> lshift;              // rows covered by one warp-wide load
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int sub = lane & (L - 1), rsel = lane >> lshift;
  const long long H = min((long long)(GT_HOT_BYTES / 16) >> lshift, rows);   // rows of the table that fit the staging buffer
  float4* __restrict__ o4 = reinterpret_cast<float4*>(out + p.col_off[t]);
  const long long ld4 = out_ld >> 2;
  const int steps = 32 / R;                // warp-wide loads to cover 32 rows

  long long rid[GT_CTA_CHUNKS];
  int n_hot = 0;
#pragma unroll
  for (int ch = 0; ch < GT_CTA_CHUNKS; ++ch) {
    const long long i = (long long)blockIdx.x * GT_CTA_ROWS + (ch * (GT_THREADS / 32) + warp) * 32 + lane;
    rid[ch] = -1;
    if (i < n) { const long long r = (long long)ids[i]; rid[ch] = (r >= 0 && r < rows) ? r : -1; }
    n_hot += (rid[ch] >= 0 && rid[ch] < H) ? 1 : 0;
  }
  if (threadIdx.x == 0) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"((uint32_t)__cvta_generic_to_shared(&hot_bar)));
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  // __syncthreads_count counts the THREADS that hold at least one hot id: a lower bound of the hits, good enough for the
  // decision (stage when the hits clearly outnumber half of the H rows the copy costs)
  n_hot = __syncthreads_count(n_hot);
  const bool staged = (long long)n_hot > H / 2 && H > 0;
  if (staged) {
    const uint32_t bar = (uint32_t)__cvta_generic_to_shared(&hot_bar);
    if (threadIdx.x == 0) {
      const uint32_t bytes = (uint32_t)(H << lshift) * 16u;
      asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
      asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                   ::"r"((uint32_t)__cvta_generic_to_shared(hot)), "l"(table), "r"(bytes), "r"(bar) : "memory");
    }
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "GT_WAIT:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], 0;\n"
        "@p bra GT_DONE;\n"
        "bra GT_WAIT;\n"
        "GT_DONE:\n"
        "}\n" ::"r"(bar) : "memory");
  }
#pragma unroll
  for (int ch = 0; ch < GT_CTA_CHUNKS; ++ch) {
    const long long i0 = (long long)blockIdx.x * GT_CTA_ROWS + (ch * (GT_THREADS / 32) + warp) * 32;
    if (i0 >= n) continue;                 // warp-uniform
    const bool lane_valid = i0 + lane < n;
    for (int s0 = 0; s0 < steps; s0 += 8) {
      float4 v[8]; bool ok[8];
#pragma unroll
      for (int u = 0; u < 8; ++u) {
        const int j = (s0 + u) * R + rsel;   // row of the chunk this lane serves in step s0+u
        const long long r = __shfl_sync(0xffffffffu, rid[ch], j & 31);
        const bool in = __shfl_sync(0xffffffffu, (int)lane_valid, j & 31) != 0;
        ok[u] = (s0 + u) < steps && in;
        if (ok[u] && r >= 0) v[u] = (staged && r < H) ? hot[(r << lshift) + sub] : __ldg(table + r * L + sub);
        else v[u] = make_float4(0.f, 0.f, 0.f, 0.f);
      }
#pragma unroll
      for (int u = 0; u < 8; ++u) {
        const int j = (s0 + u) * R + rsel;
        if (ok[u]) o4[(i0 + j) * ld4 + sub] = v[u];
      }
    }
  }
}


}  // namespace tfrs
using namespace tfrs;

extern "C" int tfrs_gather_f32(const float* const* tables, const int64_t* rows, const int32_t* dims, int n_tables,
                               const void* const* ids, int ids_dtype, int64_t n, float* out, int64_t out_ld,
                               const int32_t* out_col_off, void* stream) {
  TFRS_CHECK_ARG(n_tables > 0 && tables && rows && dims && ids && out_col_off, "gather: NULL argument");
  TFRS_CHECK_ARG(ids_dtype == TFRS_I32 || ids_dtype == TFRS_I64, "gather: ids_dtype must be I32 or I64");
  TFRS_CHECK_ARG(n >= 0 && out_ld > 0, "gather: bad n / out_ld");
  if (n == 0) return TFRS_OK;  // an empty batch: the output (and every id array) may be NULL, as empty tensors are
  TFRS_CHECK_ARG(out, "gather: NULL output");
  cudaStream_t st = (cudaStream_t)stream;
  for (int t0 = 0; t0 < n_tables; t0 += GT_MAX_TABLES) {
    int nt = n_tables - t0 < GT_MAX_TABLES ? n_tables - t0 : GT_MAX_TABLES;
    GatherParams p;
    bool vec = (out_ld % 4 == 0) && ((reinterpret_cast<uintptr_t>(out) & 15) == 0);
    int max_dim = 0;
    for (int t = 0; t < nt; ++t) {
      TFRS_CHECK_ARG(tables[t0 + t] && ids[t0 + t] && dims[t0 + t] > 0 && rows[t0 + t] >= 0, "gather: bad table %d", t0 + t);
      TFRS_CHECK_ARG(out_col_off[t0 + t] >= 0 && out_col_off[t0 + t] + dims[t0 + t] <= out_ld,
                     "gather: table %d columns [%d,%d) exceed out_ld=%lld", t0 + t, out_col_off[t0 + t],
                     out_col_off[t0 + t] + dims[t0 + t], (long long)out_ld);
      p.table[t] = tables[t0 + t]; p.ids[t] = ids[t0 + t]; p.rows[t] = rows[t0 + t];
      p.dim[t] = dims[t0 + t]; p.col_off[t] = out_col_off[t0 + t];
      vec = vec && (dims[t0 + t] % 4 == 0) && (out_col_off[t0 + t] % 4 == 0) &&
            ((reinterpret_cast<uintptr_t>(tables[t0 + t]) & 15) == 0);
      if (dims[t0 + t] > max_dim) max_dim = dims[t0 + t];
    }
    long long items = n * (vec ? max_dim / 4 : max_dim);
    long long blocks = ceil_div(items, (long long)GT_THREADS * GT_ROWS_PER_THREAD);
    if (blocks < 1) blocks = 1;
    if (blocks > 1 << 20) blocks = 1 << 20;
    dim3 grid((unsigned)blocks, (unsigned)nt);
    bool chunkable = vec;
    for (int t = 0; t < nt && chunkable; ++t) {
      const int L = p.dim[t] / 4;
      chunkable = L >= 1 && L <= 32 && (L & (L - 1)) == 0;
    }
    if (chunkable) {
      dim3 g2((unsigned)ceil_div(n, (long long)GT_CTA_ROWS), (unsigned)nt);  // GT_CTA_CHUNKS x 32 rows per warp, 8 warps per CTA
      if (ids_dtype == TFRS_I32) gather_warpchunk_kernel<int32_t><<<g2, GT_THREADS, 0, st>>>(p, n, out, out_ld);
      else gather_warpchunk_kernel<int64_t><<<g2, GT_THREADS, 0, st>>>(p, n, out, out_ld);
      TFRS_LAUNCH_CHECK();
      continue;
    }
    if (ids_dtype == TFRS_I32) {
      if (vec) gather_kernel<int32_t, true><<<grid, GT_THREADS, 0, st>>>(p, n, out, out_ld);
      else gather_kernel<int32_t, false><<<grid, GT_THREADS, 0, st>>>(p, n, out, out_ld);
    } else {
      if (vec) gather_kernel<int64_t, true><<<grid, GT_THREADS, 0, st>>>(p, n, out, out_ld);
      else gather_kernel<int64_t, false><<<grid, GT_THREADS, 0, st>>>(p, n, out, out_ld);
    }
    TFRS_LAUNCH_CHECK();
  }
  return TFRS_OK;
}
