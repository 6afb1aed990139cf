// adagrad.cuh -- K4's id grouping and argument checks, shared by every sparse optimizer step (SGD, Adagrad,
// ClippyAdagrad, Adam, FTRL), and K4's run-summing pattern with a pluggable epilogue (ClippyAdagrad's pass A, Adam, FTRL).
// K4 itself keeps its fused kernels ag_apply / ag_apply_long in adagrad.cu: instantiated from these templates, its warp
// kernel measured 0.7 us (7 %) slower on uniform cfg3 batches, about 2 % of the step (H100, BASELINE.md).
//   ag_check_args: the argument checks of the five sparse entry points (adagrad.cu)
//   ag_group:      keys = (id << 24 | position), grouped by id with positions ascending (adagrad.cu)
//   ag_run_sums:   one warp per run of equal ids (one CTA per run longer than AG_LONG) sums the run's gradient rows in
//                  order of occurrence and hands every column's sum to an epilogue op:
//                    op.column(state, row, head, d, c, g)  per column c of the run of table row `row` (element offset
//                                                          row = id * d) whose first sorted slot is `head`
//                    op.finish(state)                       once per run, reached by every thread of the warp / CTA
#pragma once
#include "common.cuh"

namespace tfrs {

constexpr unsigned long long AG_BAD_ID = 0xFFFFFFFFFFull;   // out-of-range ids sort last and are skipped

struct AgGroups {
  unsigned long long* keys;     // n sorted keys (id << 24 | position)
  unsigned int* long_count;     // runs longer than AG_LONG, queued for the CTA-per-run kernel
  unsigned int* long_list;
};
// The checks every sparse step makes before its first launch; each message starts with `who`.  `state` is false when the
// table or one of its slots is NULL.  n < 2^24 and rows < 2^40: the key holds a 24-bit position and a 40-bit id.
int ag_check_args(const char* who, bool state, long long rows, int d, int ids_dtype, long long n, const void* ids,
                  const void* grad);
size_t ag_group_workspace_bytes(long long n);
// ws must hold ag_group_workspace_bytes(n) bytes; n >= 1, ids_dtype TFRS_I32 / TFRS_I64
int ag_group(const void* ids, int ids_dtype, long long n, long long rows, void* ws, cudaStream_t st, AgGroups* out);
// The bitonic branch of ag_group on its own: the first n keys at ws come out in ascending (id, position) order, i.e. the
// groups in ascending id order as well (tree_ah.cu's leaf-major layout needs that global order).
int ag_sort(const void* ids, int ids_dtype, long long n, long long rows, void* ws, cudaStream_t st);

// Whether sorted slot i (< n) is the first slot of a run of an in-range id; the id comes back in `id`.
__device__ __forceinline__ bool ag_run_head(const unsigned long long* __restrict__ keys, long long i, unsigned long long& id) {
  id = keys[i] >> 24;
  return id != AG_BAD_ID && (i == 0 || (keys[i - 1] >> 24) != id);
}

// One warp per run of equal ids (the warp of the run's first slot; the others exit).  Duplicates are summed in order of
// occurrence -- the keys are sorted by (id, position) -- with the gradient rows of 8 members in flight per step, so a hot
// id's chain costs one DRAM round trip per 8 members instead of two per member.  Runs longer than AG_LONG members are left
// to ag_sum_runs_long (a whole CTA stages their rows through shared memory).
constexpr int AG_LONG = 64;

template <class Op>
__global__ void __launch_bounds__(256)
ag_sum_runs(const unsigned long long* __restrict__ keys, long long n, const float* __restrict__ grad, int d, const Op op,
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
  typename Op::State st{};
  const long long row = (long long)id * d;
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
    op.column(st, row, i, d, c, g);
  }
  op.finish(st);
}

// Hot ids (Zipf batches: one id can own a tenth of the batch): one CTA per long run.  All 256 threads stream the run's
// gradient rows into a shared-memory tile (AL_ROWS rows in flight per step), then one thread per column adds the tile's
// rows IN ORDER -- the chain is fp32 adds on shared memory, not DRAM round trips.
constexpr int AL_THREADS = 256, AL_ROWS = 256;  // rows per tile: min(AL_ROWS, 64 KB / row bytes)
template <class Op>
__global__ void __launch_bounds__(AL_THREADS)
ag_sum_runs_long(const unsigned long long* __restrict__ keys, long long n, const float* __restrict__ grad, int d, const Op op,
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
    typename Op::State st{};
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int c = threadIdx.x + AL_THREADS * u;
      if (c < d) op.column(st, (long long)id * d, i, d, c, acc_g[u]);
    }
    op.finish(st);
    __syncthreads();
  }
}

// The two apply launches over the grouped keys of ag_group; d <= 1024.
template <class Op>
int ag_run_sums(const AgGroups& gr, long long n, const float* grad, int d, const Op& op, cudaStream_t st) {
  TFRS_CUDA(cudaMemsetAsync(gr.long_count, 0, 4, st));
  ag_sum_runs<Op><<<(unsigned)ceil_div(n * 32, 256), 256, 0, st>>>(gr.keys, n, grad, d, op, gr.long_count, gr.long_list);
  TFRS_LAUNCH_CHECK();
  int tile_rows = (64 * 1024) / (d * 4); if (tile_rows > AL_ROWS) tile_rows = AL_ROWS; if (tile_rows < 1) tile_rows = 1;
  TFRS_DYN_SMEM(ag_sum_runs_long<Op>, 64 * 1024);
  ag_sum_runs_long<Op><<<(unsigned)sm_count(), AL_THREADS, (size_t)tile_rows * d * 4, st>>>(gr.keys, n, grad, d, op, gr.long_count,
                                                                                        gr.long_list, tile_rows);
  TFRS_LAUNCH_CHECK();
  return TFRS_OK;
}

}  // namespace tfrs
