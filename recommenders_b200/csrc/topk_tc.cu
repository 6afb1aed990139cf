// topk_tc.cu -- K2: brute-force top-K on the Hopper tensor cores (wgmma + bulk-TMA + mbarrier), sm_90a.
//
// Replaces  scores = matmul(q, c^T); top_k(scores, k)  (layers/factorized_top_k.py:603-605) for large
// corpora.  The [Q,N] score matrix never exists in HBM:
//
//   index time   tfrs_index_build : corpus fp32 -> fp16 image (exact 2^e rescale), pre-tiled as 128-row UMMA SWIZZLE_128B
//                K-major tiles (one contiguous 16 KB block per 64-wide K slab), + max row norm (scaled units).
//   query time   (0) tc_qprep     : ONE kernel, a warp per query: per-ROW power-of-two rescale (scores of different
//                    queries are never compared, so every query gets its own exponent), fp16 tile image, error margins
//                (1) tc_scan<SAMPLE> : screening GEMM over every 4th corpus tile (or, on an index that chose it, the
//                    highest-norm eighth of the corpus, see SAMPLE_NORM); each epilogue thread keeps the maximum
//                    of a GROUP of tiles (a "bin") -> <= 1024 bins per query; tc_threshold (a warp per query, bins in
//                    registers) takes the K-th largest bin maximum L_q: K distinct bins hold K distinct candidates
//                    >= L_q, so L_q is a valid lower bound of the K-th best screening score; top-K and EXCLUDE calls
//                    filter at the K'-th largest (filter_bin_rank, K' < K: a bound but for ~1e-9 of rows in random
//                    order) and keep L_q for the rows that miss, which are filtered and selected again (retry)
//                (2) tc_scan<FILTER> : screening GEMM over the whole corpus; epilogue compares the fp32
//                    accumulators (in registers) with T_q = L_q - margin_q and appends the rare
//                    survivors (octet records) to per-(query, part, half) lists -- nothing else leaves the SM
//                (3) tc_finalize (a warp per query, no block barriers): tau = K-th best screening score; survivors
//                    within the error band of tau are re-scored EXACTLY (sequential fp32 fmaf chain on the fp32
//                    corpus) and ranked by (score desc, index asc) -> bit-identical to the exact CUDA-core path.
//                    Variants of the same kernel: EXCLUDE (query_with_exclusions, :83-115,242-288: the k+E best are
//                    re-ranked with excluded identifiers lowered by 1e5) and COUNT (the FactorizedTopK metric,
//                    metrics/factorized_top_k.py:133-192: #{candidates scoring above the positive}, no top-K list).
//                (4) overflow fallback (list capacity exceeded; adversarial inputs only): exact scan.
//
// Why the result is exact: |screen(q,c) - exact(q,c)| <= eps_q = E_REL*|q|*max|c| (fp16 rounding of both
// operands: (2u+u^2) sum|q_k c_k| with u = 2^-11, plus accumulation slack; Cauchy-Schwarz).  Any member
// of the exact top-K has screening score >= tau - 2*eps_q >= L_q - 2*eps_q, so it is in the list and in
// the re-scored band.
//
// Scan kernel shape (per CTA, 1 CTA / SM, 512 threads = 16 warps, so 128 registers per thread): 256 queries (two
// 128-row A blocks) x a contiguous range of 128-row corpus tiles streamed through a 4-6 stage bulk-TMA ring, which
// thread 0 drives between its own MMAs.  Warpgroups 0-3 own one 64-query slice each and run every tile as two
// 64-column halves (wgmma m64n64k16, fp16 -> fp32 in two 32-register accumulator sets): the MMAs of the next half are
// in flight while the epilogue of the current one runs, so no warpgroup waits for its own MMAs before its epilogue.
// For d <= 64 a warpgroup's A slice lives in registers (RS wgmma, half the smem reads of SS); for d <= 128 it stays in
// smem.  Each B tile in smem feeds all four (256 query rows per 16 KB of L2->smem traffic).
#include <cuda_fp16.h>
#include <math.h>
#include <stdlib.h>
#include <type_traits>
#include "rowselect.cuh"
#include "tc_ptx.cuh"

namespace tfrs {
namespace tc {

constexpr int TILE_N = 128;          // corpus rows per B tile
constexpr int TILE_M = 128;          // query rows per A block
constexpr int QBLK = 256;            // queries per CTA (2 A blocks)
constexpr int KSLAB = 64;            // fp16 elements per 128-byte swizzle row
constexpr int SLAB_BYTES = TILE_N * 128;  // 16 KB: 128 rows x 128 B
constexpr int HEADER_BYTES = 1024;
constexpr int THREADS = 512;         // 4 consumer warpgroups (16 warps: 128 registers per thread)
constexpr int CONSUMER_WARPS = 16;
constexpr int CAND_CAP = 2048;       // octet records kept per query across all segments (sizing of cap_part)
constexpr int MAX_SAMPLE_STRIDE = 4;
constexpr int FIN_MAX_PARTS = 2 * 132;  // survivor-list segments per query: (corpus part, column half); parts <= SMs
constexpr int MAX_BINS = 1024;       // bin maxima per query (32 per lane of the threshold warp)
constexpr int FP16_TARGET = 15;      // largest operand magnitude lands in [2^14, 2^15)
// Screening error model (operands: fp16 after an exact power-of-two rescale -- one exponent for the whole corpus,
// one per query row -- so that the largest magnitude lands in [2^14, 2^15); accumulate: fp32 in registers):
//   |x^ - x| <= 2^-11 |x| (+2^-25 absolute below the fp16 normal range, negligible after the rescale)
//   => |screen - exact| <= (2^-10 + 2^-22) sum|q_k c_k|  + accumulation slack (budget 2^-14) + fmaf-chain 2^-16
//   <= E_REL * |q| * |c|   (Cauchy-Schwarz), E_REL = 0.00108 including the 0.1 % norm inflation.
constexpr float E_REL = 0.00108f;
constexpr float E_ACC = 0.00013f;    // run-to-run slack between the two passes (they are bit-identical in practice)

struct SideStats {              // corpus side, written at index time
  unsigned int max_norm2_bits;  // max_i |x_i * 2^exp|^2  (SCALED units; float bits; non-negative so uint order == float order)
  unsigned int amax_bits;       // max_ij |x_ij|
  int exp;                      // rescale exponent e: x * 2^e has its largest magnitude in [2^14, 2^15)
  int pad;
};
// Sample of the sampled pass, chosen per index at build time (tfrs_index_build):
//   SAMPLE_STRIDED  every stride-th tile of the corpus image (Plan::stride)
//   SAMPLE_NORM     the norm-sample image: the floor(N/8) rows of largest norm (rounded down to whole tiles), in index
//                   order, stored after the corpus image.  Winners of a dot-product top-K have above-average norms, so
//                   half the strided sample's rows give as tight a k-th bin bound.  Taken when N >= 2^19 and both
//                   (a) the random-direction model (norm_phi_*) gives the sample phi >= 0.35 of the expected top 1e-4;
//                   (b) probe queries made of corpus rows find their neighbours in the sample: the model cannot see
//                       queries that align with groups of rows (a clustered corpus, whose high-norm clusters are not
//                       every query's own), where the sample's bound is loose and rows would take the exact fallback.
//                       NORM_PROBES evenly spaced rows, each scored against the corpus (the exact top-(K+1) of the
//                       strided-sample path, itself dropped): the share of each probe's K neighbours that lie in the
//                       sample must average >= 0.35 and be >= 0.25 (the strided sample's own share) for every probe.
// The choice is made once, at build; a query call never writes the index.
enum { SAMPLE_STRIDED = 0, SAMPLE_NORM = 1 };
constexpr long long NORM_SAMPLE_MIN_N = 1ll << 19;   // below this the sample's tiles cannot fill the bins
constexpr int NORM_SAMPLE_DIV = 8;                   // sample rows = N / 8
constexpr double NORM_SAMPLE_TAIL = 1e-4;            // phi is measured on the expected top N * 1e-4 scores
constexpr double NORM_SAMPLE_MIN_PHI = 0.35;
constexpr int NORM_PROBES = 256, NORM_PROBE_K = 100;
constexpr float NORM_PROBE_MIN_MEAN = 0.35f, NORM_PROBE_MIN_EACH = 0.25f;
struct IndexHeader {
  SideStats st;
  int d, d_pad, kb, sample;   // sample: SAMPLE_STRIDED / SAMPLE_NORM
  long long n, n_tiles;
  float phi;                  // the norm sample's phi (0 below NORM_SAMPLE_MIN_N)
  float probe_mean, probe_min;   // the probes' neighbour share in the sample (0 below NORM_SAMPLE_MIN_N)
};
// tiles of the norm-sample image of an N-row corpus (0: the index has none)
__host__ __device__ inline long long norm_sample_tiles(long long N) {
  return N >= NORM_SAMPLE_MIN_N && N < (1ll << 31) ? N / NORM_SAMPLE_DIV / 128 : 0;
}

__device__ __forceinline__ int rescale_exp(float amax) {
  int x = 0;
  if (!(amax > 0.f) || !(amax < INFINITY)) return 0;
  (void)frexpf(amax, &x);      // amax = m * 2^x, m in [0.5, 1)
  return FP16_TARGET - x;      // amax * 2^exp in [2^(target-1), 2^target)
}

// ------------------------------------------------------------------------------------------------
// image builders: fp32 [rows, d] -> fp16 128-row tiles, each K slab of 64 as one swizzled 16 KB block
//   byte offset of element (r, k) inside a tile = (k/64)*16384 + r*128 + (((k%64)/8) ^ (r%8))*16 + (k%8)*2
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
tile_image_kernel(const float* __restrict__ src, long long rows, int d, int kb, long long n_tiles,
                  const SideStats* __restrict__ st, unsigned char* __restrict__ img, const int* __restrict__ rowmap) {
  // rowmap (norm-sample image): image row i holds corpus row rowmap[i], with the same bits as in the corpus image
  const int scale_exp = st->exp;
  const long long total = n_tiles * TILE_N * (long long)kb * 8;  // 16-byte chunks
  for (long long e = (long long)blockIdx.x * 256 + threadIdx.x; e < total; e += (long long)gridDim.x * 256) {
    int chunk = (int)(e % (kb * 8));
    long long row = e / (kb * 8);
    int slab = chunk / 8, cj = chunk % 8;
    int r = (int)(row % TILE_N);
    long long tile = row / TILE_N;
    int k0 = slab * KSLAB + cj * 8;
    const long long srow = (rowmap != nullptr && row < rows) ? (long long)rowmap[row] : row;
    __align__(16) __half v[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      float f = (row < rows && k0 + j < d) ? src[srow * d + k0 + j] : 0.f;
      v[j] = __float2half_rn(ldexpf(f, scale_exp));  // exact power-of-two rescale, then one rounding to fp16
    }
    unsigned char* dst = img + tile * ((long long)kb * SLAB_BYTES) + (long long)slab * SLAB_BYTES + r * 128 + ((cj ^ (r & 7)) * 16);
    *reinterpret_cast<uint4*>(dst) = *reinterpret_cast<const uint4*>(v);
  }
}

// corpus statistics, two passes (one warp per row -> coalesced): PASS 0 max |element| -> exponent; PASS 1 max row norm^2
// of the SCALED rows (so tiny or huge corpora neither underflow nor overflow the fp32 norm)
template <int PASS>
__global__ void __launch_bounds__(256)
corpus_stats_kernel(const float* __restrict__ src, long long rows, int d, SideStats* __restrict__ st,
                    unsigned int* __restrict__ norm2_key = nullptr) {   // PASS 1: each row's scaled norm^2 (float bits)
  const int lane = threadIdx.x & 31;
  const long long warp = ((long long)blockIdx.x * 256 + threadIdx.x) >> 5;
  const long long nwarps = ((long long)gridDim.x * 256) >> 5;
  const int e = PASS ? st->exp : 0;
  float best = 0.f;
  for (long long row = warp; row < rows; row += nwarps) {
    const float* p = src + row * d;
    float acc = 0.f;
    for (int k = lane; k < d; k += 32) {
      const float x = p[k];
      if (PASS) { const float y = ldexpf(x, e); acc = fmaf(y, y, acc); } else acc = fmaxf(acc, fabsf(x));
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float other = __shfl_xor_sync(0xffffffffu, acc, o);
      acc = PASS ? acc + other : fmaxf(acc, other);
    }
    if (PASS && norm2_key != nullptr && lane == 0) norm2_key[row] = __float_as_uint(acc);   // >= 0: uint order == float order
    best = fmaxf(best, acc);
  }
  if (lane == 0 && best > 0.f) {
    if (PASS) atomicMax(&st->max_norm2_bits, __float_as_uint(best * 1.0001f));  // slack for the tree order
    else atomicMax(&st->amax_bits, __float_as_uint(best));
  }
}
__global__ void side_exp_kernel(SideStats* st) { st->exp = rescale_exp(__uint_as_float(st->amax_bits)); }
__global__ void header_kernel(IndexHeader* dst, IndexHeader h) { *dst = h; }

// ---- norm sample (index time, all on the device; every reduction in a fixed order, so the index is deterministic) ----
// State of the build in scratch memory.  The S-th largest norm key T is found bit by bit, from the top: cnt[b] =
// #{key >= prefix | 2^b} with the bits above b decided by cnt[31..b+1] (norm_select_prefix), so one kernel per bit.
struct NormSelect {
  unsigned long long cnt[32];
  long long need;      // rows with key == T that join the sample (the lowest indices among them)
  double lo, hi;       // bisection bracket of the tail point t (norm_phi_*)
};
constexpr int NS_CHUNK = 8192;   // rows per block in the compaction and the phi sums (256 threads x 32)

__device__ __forceinline__ unsigned int norm_select_prefix(const NormSelect* s, long long S, int lowest) {
  unsigned int prefix = 0u;
  for (int b = 31; b > lowest; --b)
    if (s->cnt[b] >= (unsigned long long)S) prefix |= 1u << b;
  return prefix;
}

__global__ void __launch_bounds__(256)
norm_select_count_kernel(const unsigned int* __restrict__ key, long long n, long long S, int bit, NormSelect* s) {
  const unsigned int cand = norm_select_prefix(s, S, bit) | (1u << bit);
  unsigned int c = 0;
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < n; i += (long long)gridDim.x * 256) c += key[i] >= cand ? 1u : 0u;
  c = __reduce_add_sync(0xffffffffu, c);
  if ((threadIdx.x & 31) == 0 && c) atomicAdd(&s->cnt[bit], (unsigned long long)c);
}

// per chunk: #{key > T}, #{key == T}
__global__ void __launch_bounds__(256)
norm_select_chunks_kernel(const unsigned int* __restrict__ key, long long n, long long S, const NormSelect* s, int* __restrict__ blk) {
  __shared__ int sh[2];
  const unsigned int T = norm_select_prefix(s, S, -1);
  if (threadIdx.x == 0) { sh[0] = 0; sh[1] = 0; }
  __syncthreads();
  int gt = 0, eq = 0;
  const long long r0 = (long long)blockIdx.x * NS_CHUNK;
  for (int t = threadIdx.x; t < NS_CHUNK; t += 256) {
    const long long i = r0 + t;
    if (i < n) { gt += key[i] > T ? 1 : 0; eq += key[i] == T ? 1 : 0; }
  }
  gt = __reduce_add_sync(0xffffffffu, gt); eq = __reduce_add_sync(0xffffffffu, eq);
  if ((threadIdx.x & 31) == 0) { atomicAdd(&sh[0], gt); atomicAdd(&sh[1], eq); }
  __syncthreads();
  if (threadIdx.x == 0) { blk[2 * blockIdx.x] = sh[0]; blk[2 * blockIdx.x + 1] = sh[1]; }
}

// one thread: chunk counts -> each chunk's first sample position and first tie rank (in place), and `need`
__global__ void norm_select_offsets_kernel(int* __restrict__ blk, int nblk, long long S, NormSelect* s) {
  long long gt = 0;
  for (int b = 0; b < nblk; ++b) gt += blk[2 * b];
  const long long need = S - gt;
  long long sel = 0, eq = 0;
  for (int b = 0; b < nblk; ++b) {
    const long long g = blk[2 * b], e = blk[2 * b + 1];
    const long long take = need - eq < 0 ? 0 : (need - eq < e ? need - eq : e);
    blk[2 * b] = (int)sel; blk[2 * b + 1] = (int)eq;
    sel += g + take; eq += e;
  }
  s->need = need;
}

// stable compaction: rowlist[] = the rows with key > T and the first `need` rows with key == T, in index order
__global__ void __launch_bounds__(256)
norm_select_write_kernel(const unsigned int* __restrict__ key, long long n, long long S, const NormSelect* s,
                         const int* __restrict__ blk, int* __restrict__ rowlist) {
  __shared__ int wsel[8], weq[8];
  const unsigned int T = norm_select_prefix(s, S, -1);
  const long long need = s->need;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const unsigned int lt = (1u << lane) - 1u;
  int sel_base = blk[2 * blockIdx.x], eq_base = blk[2 * blockIdx.x + 1];
  const long long r0 = (long long)blockIdx.x * NS_CHUNK;
  for (int t0 = 0; t0 < NS_CHUNK; t0 += 256) {
    const long long i = r0 + t0 + threadIdx.x;
    const unsigned int k = i < n ? key[i] : 0u;
    const bool is_eq = i < n && k == T;
    const unsigned int veq = __ballot_sync(0xffffffffu, is_eq);
    if (lane == 0) weq[warp] = __popc(veq);
    __syncthreads();
    int eq_before = eq_base, eq_all = 0;
    for (int w = 0; w < 8; ++w) { eq_before += w < warp ? weq[w] : 0; eq_all += weq[w]; }
    eq_before += __popc(veq & lt);
    const bool is_sel = i < n && (k > T || (is_eq && eq_before < need));
    const unsigned int vsel = __ballot_sync(0xffffffffu, is_sel);
    if (lane == 0) wsel[warp] = __popc(vsel);
    __syncthreads();
    int sel_before = sel_base, sel_all = 0;
    for (int w = 0; w < 8; ++w) { sel_before += w < warp ? wsel[w] : 0; sel_all += wsel[w]; }
    if (is_sel) rowlist[sel_before + __popc(vsel & lt)] = (int)i;
    sel_base += sel_all; eq_base += eq_all;
    __syncthreads();
  }
}

// Random-direction model: a row of norm r scores r g, g ~ N(0, 1), so it exceeds t with probability erfc(t / (r sqrt 2)) / 2.
// t solves sum_i P_i(t) = N * NORM_SAMPLE_TAIL (bisection); phi = sum over the sample of P_i(t) / (N * NORM_SAMPLE_TAIL).
__device__ __forceinline__ double norm_tail(unsigned int norm2_key, double t) {
  const double r = sqrt((double)__uint_as_float(norm2_key));
  return r > 0.0 ? 0.5 * erfc(t / (r * 1.4142135623730951)) : 0.0;
}
// per chunk: sum of P_i(t) at the bracket's midpoint over key[rows[j]] (rows == nullptr: key[j]), j < n; fixed order
__global__ void __launch_bounds__(256)
norm_phi_partial_kernel(const unsigned int* __restrict__ key, const int* __restrict__ rows, long long n, const NormSelect* s,
                        double* __restrict__ partial) {
  __shared__ double sh[256];
  const double t = 0.5 * (s->lo + s->hi);
  double acc = 0.0;
  const long long r0 = (long long)blockIdx.x * NS_CHUNK;
  for (int u = threadIdx.x; u < NS_CHUNK; u += 256) {
    const long long j = r0 + u;
    if (j < n) acc += norm_tail(key[rows ? (long long)rows[j] : j], t);
  }
  sh[threadIdx.x] = acc;
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if (threadIdx.x < o) sh[threadIdx.x] += sh[threadIdx.x + o];
    __syncthreads();
  }
  if (threadIdx.x == 0) partial[blockIdx.x] = sh[0];
}
// one thread.  final == 0: one bisection step;  final == 1: the sample's sum -> phi, and with the probes' neighbour
// shares (share[NORM_PROBES]) the header's choice
__global__ void norm_phi_step_kernel(const double* __restrict__ partial, int nblk, long long N, int final, NormSelect* s,
                                     IndexHeader* hdr, const float* __restrict__ share) {
  double sum = 0.0;
  for (int b = 0; b < nblk; ++b) sum += partial[b];
  const double target = (double)N * NORM_SAMPLE_TAIL;
  if (!final) {
    const double t = 0.5 * (s->lo + s->hi);
    if (sum > target) s->lo = t; else s->hi = t;
  } else {
    const double phi = sum / target;
    float mean = 0.f, mn = 1.f;
    for (int i = 0; i < NORM_PROBES; ++i) { mean += share[i]; mn = fminf(mn, share[i]); }
    mean /= NORM_PROBES;
    hdr->phi = (float)phi; hdr->probe_mean = mean; hdr->probe_min = mn;
    // NaN (non-finite rows) fails every comparison: strided
    hdr->sample = phi >= NORM_SAMPLE_MIN_PHI && mean >= NORM_PROBE_MIN_MEAN && mn >= NORM_PROBE_MIN_EACH ? SAMPLE_NORM : SAMPLE_STRIDED;
  }
}

// probe p = corpus row p * N / NORM_PROBES; one warp per probe row: its fp32 copy
__global__ void norm_probe_gather_kernel(const float* __restrict__ corpus, long long N, int d, float* __restrict__ probes) {
  const int pr = blockIdx.x;
  const long long row = (long long)pr * N / NORM_PROBES;
  for (int t = threadIdx.x; t < d; t += 32) probes[(long long)pr * d + t] = corpus[row * d + t];
}
// in_sample[row] = 1 for the sample's rows
__global__ void norm_sample_flags_kernel(const int* __restrict__ rowlist, long long S, unsigned char* __restrict__ in_sample) {
  for (long long j = (long long)blockIdx.x * 256 + threadIdx.x; j < S; j += (long long)gridDim.x * 256) in_sample[rowlist[j]] = 1;
}
// one warp per probe: the share of its K best neighbours (the top K + 1 without the probe's own row) in the sample
__global__ void norm_probe_share_kernel(const long long* __restrict__ idx, long long N, const unsigned char* __restrict__ in_sample,
                                        float* __restrict__ share) {
  const int pr = blockIdx.x, lane = threadIdx.x;
  const long long self = (long long)pr * N / NORM_PROBES;
  int hit = 0, n = 0;
  for (int j = lane; j < NORM_PROBE_K + 1; j += 32) {
    const long long i = idx[(long long)pr * (NORM_PROBE_K + 1) + j];
    if (i != self && i >= 0 && i < N) { ++n; hit += in_sample[i]; }
  }
  hit = __reduce_add_sync(0xffffffffu, hit); n = __reduce_add_sync(0xffffffffu, n);
  if (lane == 0) share[pr] = n > 0 ? (float)hit / (float)n : 0.f;
}
__global__ void norm_phi_init_kernel(NormSelect* s, const SideStats* st) {
  s->lo = 0.0;
  s->hi = 40.0 * sqrt((double)__uint_as_float(st->max_norm2_bits)) + 1e-30;   // P <= erfc(28) ~ 1e-343 per row above it
}

// (0) query preparation, one warp per (padded) query row: per-row exponent, scaled norm -> margins, fp16 tile image.
//   margin[row] = 2*eps + run-to-run slack  (filter threshold T = L - margin)
//   cut[row]    = 2*eps                      (band below tau that is re-scored exactly)
//   qexp[row]   = the row's exponent (COUNT mode converts the positive score to screening units with it)
// All in SCREENING units: scores scaled by 2^(exp_corpus + exp_row), an exact power of two.
__global__ void __launch_bounds__(256)
tc_qprep_kernel(const float* __restrict__ q, long long Q, long long Qp, int d, int kb, const IndexHeader* __restrict__ hdr,
                unsigned char* __restrict__ qimg, float* __restrict__ margin, float* __restrict__ cut, int* __restrict__ qexp) {
  const int lane = threadIdx.x & 31;
  const long long row = ((long long)blockIdx.x * 256 + threadIdx.x) >> 5;
  if (row >= Qp) return;
  const bool real = row < Q;
  const float* p = q + row * d;
  float a = 0.f;
  if (real) for (int k = lane; k < d; k += 32) a = fmaxf(a, fabsf(p[k]));
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) a = fmaxf(a, __shfl_xor_sync(0xffffffffu, a, o));
  const int e = rescale_exp(a);
  float n2 = 0.f;
  if (real) for (int k = lane; k < d; k += 32) { const float y = ldexpf(p[k], e); n2 = fmaf(y, y, n2); }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) n2 += __shfl_xor_sync(0xffffffffu, n2, o);
  if (lane == 0) {
    const float cn = sqrtf(__uint_as_float(hdr->st.max_norm2_bits)) * 1.001f;   // scaled corpus norm bound
    const float qn = sqrtf(n2 * 1.0001f) * 1.001f;                               // scaled query norm (+ tree-order slack)
    const float eps = E_REL * qn * cn + 1e-30f;
    margin[row] = 2.f * eps + E_ACC * qn * cn;
    cut[row] = 2.f * eps;
    qexp[row] = e;
  }
  // image: chunk (slab, cj) of this row; kb*8 <= 16 chunks, one lane each
  const int r = (int)(row % TILE_N);
  const long long tile = row / TILE_N;
  if (lane < kb * 8) {
    const int slab = lane >> 3, cj = lane & 7;
    const int k0 = slab * KSLAB + cj * 8;
    __align__(16) __half v[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float f = (real && k0 + j < d) ? p[k0 + j] : 0.f;
      v[j] = __float2half_rn(ldexpf(f, e));
    }
    unsigned char* dst = qimg + tile * ((long long)kb * SLAB_BYTES) + (long long)slab * SLAB_BYTES + r * 128 + ((cj ^ (r & 7)) * 16);
    *reinterpret_cast<uint4*>(dst) = *reinterpret_cast<const uint4*>(v);
  }
}

// ------------------------------------------------------------------------------------------------
// the screening GEMM
// ------------------------------------------------------------------------------------------------
enum { MODE_SAMPLE = 0, MODE_FILTER = 1 };

// A/B ablations of the FILTER pass, timed by tools/filter_probe.py.  They exist only in the debug libraries that
// `python -m recommenders_b200.build --debug-switches VARIANT` writes; the product library is always FILTER_FULL.
// A call with an ablated pass stops after it and leaves its outputs unwritten: only the stage times
// (tfrs_profile_read) mean anything.
//   FILTER_NO_EMIT      hit test and octet mask computed, nothing stored
//   FILTER_NO_EPILOGUE  the accumulators XOR-folded into one live word (ptxas deletes MMAs whose results are never read)
enum { FILTER_FULL = 0, FILTER_NO_EMIT = 1, FILTER_NO_EPILOGUE = 2 };
#if defined(TFRS_DEBUG_SWITCHES) && defined(TFRS_FILTER_ABLATION)
constexpr int FILTER_ABLATION = TFRS_FILTER_ABLATION;
#else
constexpr int FILTER_ABLATION = FILTER_FULL;
#endif

struct ScanParams {
  const unsigned char* qimg;    // query tile image  [2*nqb tiles][KB][16 KB]
  const unsigned char* cimg;    // corpus tile image [n_tiles][KB][16 KB]
  long long Q, N;
  int nqb, parts, n_seq, stride;  // tile sequence: tile(u) = u * stride, u in [0, n_seq)
  long long n_tiles;
  // SAMPLE: a bin = the maximum over `group` consecutive sampled tiles x 64 columns of one epilogue thread
  float* binmax; int bins_ld;     // [Qp, bins_ld]; bin = (part * bins_per_part + it / group) * 2 + half
  int group, bins_per_part;
  // SAMPLE on an index whose header says SAMPLE_NORM (simg != null): the norm-sample image at stride 1, same parts
  const IndexHeader* hdr;
  const unsigned char* simg;
  int n_seq_norm, group_norm, bins_per_part_norm;
  // FILTER
  const float* thr;               // [Qp]
  // Retry launch (null on the first filter pass): [Qp] marks of the rows the select kernel sends back at their guaranteed
  // threshold.  Only those rows rewrite their records and counts; a CTA whose 256 queries hold none exits at once.
  const unsigned int* retry;
  unsigned int* count;            // [Qp, parts, 2]   records written by each (query, corpus part, half)
  // Survivor RECORDS: when any of 8 consecutive columns of a row passes the threshold, the whole octet is
  // appended (two 16-byte stores + the index of its first column); finalize drops the non-survivors.
  // One private segment per (query row, corpus part, column half): a single writer thread, no atomics.
  float* cand_s;                  // [Qp, parts, 2, cap_part, 8] screening scores of the octet
  unsigned int* cand_i;           // [Qp, parts, 2, cap_part]    local index of the octet's first column
  int cap_part;                   // records per segment
};

// NORM: the sampled pass over the norm-sample image (a compile-time choice, so the strided tile sequence keeps its
// parameter reads and the code it had before the norm sample existed)
template <int KB, int STAGES, int MODE, bool NORM>
__device__ __forceinline__ void tc_scan_body(const ScanParams& p) {
  extern __shared__ __align__(1024) unsigned char smem_raw[];
  // carve: [A: 2*KB slabs][B: STAGES*KB slabs][barriers]
  unsigned char* smem = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  unsigned char* sA = smem;
  unsigned char* sB = smem + 2 * KB * SLAB_BYTES;
  uint64_t* bars = reinterpret_cast<uint64_t*>(sB + STAGES * KB * SLAB_BYTES);
  uint64_t* full = bars;                 // [STAGES]
  uint64_t* empty = bars + STAGES;       // [STAGES]
  uint64_t* a_full = bars + 2 * STAGES;  // [1]

  const int wg = threadIdx.x >> 7, warp = (threadIdx.x >> 5) & 3, lane = threadIdx.x & 31;
  const int qb = blockIdx.x % p.nqb, part = blockIdx.x / p.nqb;
  // the tile sequence: the norm-sample image at stride 1, else every stride-th tile of the corpus image
  const unsigned char* const cimg = NORM ? p.simg : p.cimg;
  const int n_seq = NORM ? p.n_seq_norm : p.n_seq, stride = NORM ? 1 : p.stride;
  const int group = NORM ? p.group_norm : p.group, bins_per_part = NORM ? p.bins_per_part_norm : p.bins_per_part;
  const int u_begin = (int)((long long)part * n_seq / p.parts);
  const int u_end = (int)((long long)(part + 1) * n_seq / p.parts);
  const int n_iter = u_end - u_begin;
  const bool issuer = threadIdx.x == 0;   // also drives the bulk-TMA ring
  // rows this launch (re)writes: every row on the first filter pass, the marked ones on a retry
  auto rescanned = [&](long long row) { return p.retry == nullptr || (row < p.Q && p.retry[row] != 0u); };
  if (MODE == MODE_FILTER && p.retry != nullptr &&
      !__syncthreads_or(threadIdx.x < QBLK && rescanned((long long)qb * QBLK + threadIdx.x)))
    return;

  if (issuer) {
    for (int s = 0; s < STAGES; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], CONSUMER_WARPS); }
    mbar_init(a_full, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  // tile `it` of this part -> ring slot `stage` (issuer only)
  auto load_tile = [&](int it, int stage) {
    const long long tile = (long long)(u_begin + it) * stride;
    mbar_expect_tx(&full[stage], KB * SLAB_BYTES);
    if (MODE == MODE_FILTER)   // streamed once per pass: evict-first, so the survivor records stay in L2 for the select kernel
      bulk_g2s_hint(sB + stage * KB * SLAB_BYTES, cimg + tile * ((long long)KB * SLAB_BYTES), KB * SLAB_BYTES, &full[stage],
                    l2_policy_evict_first());
    else
      bulk_g2s(sB + stage * KB * SLAB_BYTES, cimg + tile * ((long long)KB * SLAB_BYTES), KB * SLAB_BYTES, &full[stage]);
  };
  if (issuer) {
    mbar_expect_tx(a_full, 2 * KB * SLAB_BYTES);
    bulk_g2s(sA, p.qimg + (long long)qb * 2 * KB * SLAB_BYTES, 2 * KB * SLAB_BYTES, a_full);
    for (int it = 0; it < STAGES && it < n_iter; ++it) load_tile(it, it);
  }

  // Warpgroup wg computes the 64 query rows [64 wg, 64 wg + 64) of the CTA's 256 against each tile, as two 64-column
  // halves (m64n64k16, one 32-register accumulator set each).  The MMAs of the next half are issued before the epilogue
  // of the current one, so every warpgroup keeps the tensor pipe busy while it runs its own epilogue.  A thread holds rows
  // r and r + 8 x 16 columns of a half (pairs 8j + 2(lane%4) + {0,1}, j < 8); the 4 lanes of a quad together hold 8
  // consecutive columns of a row -- one octet record.
  const long long row_a = (long long)qb * QBLK + wg * 64 + warp * 16 + (lane >> 2);   // rows row_a, row_a + 8
  const bool quad_leader = (lane & 3) == 0;
  float thr[2] = {INFINITY, INFINITY};
  if (MODE == MODE_FILTER) {
    // a row a retry launch does not rescan gets a NaN threshold, which no score passes (not even +inf): its records stay
#pragma unroll
    for (int rr = 0; rr < 2; ++rr) if (row_a + 8 * rr < p.Q) thr[rr] = rescanned(row_a + 8 * rr) ? p.thr[row_a + 8 * rr] : NAN;
  }
  const unsigned int cap = (unsigned int)p.cap_part;
  unsigned int cnt[4] = {0u, 0u, 0u, 0u}, ovf = 0u;      // segment s = (row rr, column half h) = 2 rr + h
  unsigned int sink = 0u;                                // what an ablated FILTER epilogue keeps live
  long long seg_base[2];                                 // first record of segment (row rr, half 0); half 1 follows it
#pragma unroll
  for (int rr = 0; rr < 2; ++rr) seg_base[rr] = ((row_a + 8 * rr) * p.parts + part) * 2 * (long long)cap;
  float binm[4] = {-INFINITY, -INFINITY, -INFINITY, -INFINITY};
  int in_group = 0, bin_out = 0;

  mbar_wait(a_full, 0);
  // this warpgroup's 64-row slice of A block wg/2 (image layout [block][K slab][16 KB]): 8 swizzle groups of 1024 B
  const uint32_t a0 = smem_u32(sA + (wg >> 1) * KB * SLAB_BYTES + (wg & 1) * 8192);
  // KB == 1: the slice stays the same for the whole scan, so it lives in registers (RS wgmma), which halves the
  // shared-memory reads per MMA; one ldmatrix_x4 per K step of 16.  Lane t addresses row 16 warp + 8 ((t/8) & 1) + t%8,
  // 16-byte chunk 2 k4 + t/16 of the swizzled slice.
  uint32_t afrag[4][4];
  if (KB == 1) {
    const int r = warp * 16 + ((lane >> 3) & 1) * 8 + (lane & 7);
#pragma unroll
    for (int k4 = 0; k4 < 4; ++k4) ldmatrix_x4(afrag[k4], a0 + r * 128 + (((2 * k4 + (lane >> 4)) ^ (lane & 7)) * 16));
  }
  // the MMAs of one 64-column half of the tile in ring slot `stage`; one commit group
  auto issue = [&](float (&acc)[32], int stage, int h) {
    wgmma_fence();
#pragma unroll
    for (int kb = 0; kb < KB; ++kb) {
      const uint64_t b_desc = make_smem_desc(smem_u32(sB + (stage * KB + kb) * SLAB_BYTES + h * 8192));
#pragma unroll
      for (int k4 = 0; k4 < 4; ++k4) {  // 4 x (K=16 fp16 = 32 B) inside the 128-byte swizzle row
        if (KB == 1)
          wgmma_m64n64_rs(acc, afrag[k4], b_desc + (uint64_t)(k4 * 2), (uint32_t)(k4 != 0));
        else
          wgmma_m64n64_ss(acc, make_smem_desc(a0 + kb * SLAB_BYTES) + (uint64_t)(k4 * 2), b_desc + (uint64_t)(k4 * 2),
                          (uint32_t)((kb | k4) != 0));
      }
    }
    wgmma_commit();
  };
  // the epilogue of half H of tile `it` (first column col0)
  auto epilogue = [&](const float (&acc)[32], long long col0, int it, auto half) {
    constexpr int H = decltype(half)::value;
    if (MODE != MODE_FILTER) {
#pragma unroll
      for (int j = 0; j < 8; ++j)
#pragma unroll
        for (int rr = 0; rr < 2; ++rr) binm[2 * rr + H] = max3(binm[2 * rr + H], acc[4 * j + 2 * rr], acc[4 * j + 2 * rr + 1]);
      if (H == 1 && (++in_group == group || it == n_iter - 1)) {   // close the bin after `group` tiles (loop-uniform)
#pragma unroll
        for (int s = 0; s < 4; ++s) {
          const float m = quad_max(binm[s]);
          const long long row = row_a + 8 * (s >> 1);
          if (quad_leader && row < p.Q)
            p.binmax[row * p.bins_ld + (long long)part * bins_per_part * 2 + (s & 1) + 2 * bin_out] = m;
          binm[s] = -INFINITY;
        }
        ++bin_out; in_group = 0;
      }
    } else {
      // Common path: a max tree over each row's 16 scores, one compare per row and one warp vote.  A warp of 16 rows meets
      // a survivor in about one half tile in two.  Only then each lane marks the octets (row rr, column group j) where one
      // of its two scores passes.  An octet belongs to one row and its 8 columns to the 4 lanes of one quad, so an OR over
      // the quad (two shuffles) makes the decision quad-uniform, with no warp-wide vote: each lane of a surviving octet
      // stores its two scores, the quad leader the octet's first index, in ascending column order within the segment.
      if (FILTER_ABLATION == FILTER_NO_EPILOGUE) {   // all 32 registers read: with one, ptxas serializes the wgmma (C7511)
#pragma unroll
        for (int i = 0; i < 32; ++i) sink ^= __float_as_uint(acc[i]);
        return;
      }
      float pm[2][8];
      bool pass = false;
#pragma unroll
      for (int rr = 0; rr < 2; ++rr) {
#pragma unroll
        for (int j = 0; j < 8; ++j) pm[rr][j] = fmaxf(acc[4 * j + 2 * rr], acc[4 * j + 2 * rr + 1]);
        const float m = fmaxf(fmaxf(fmaxf(pm[rr][0], pm[rr][1]), fmaxf(pm[rr][2], pm[rr][3])),
                              fmaxf(fmaxf(pm[rr][4], pm[rr][5]), fmaxf(pm[rr][6], pm[rr][7])));
        pass |= m >= thr[rr];
      }
      if (__any_sync(0xffffffffu, pass)) {
        unsigned int mine = 0u;
#pragma unroll
        for (int rr = 0; rr < 2; ++rr)
#pragma unroll
          for (int j = 0; j < 8; ++j) mine |= (pm[rr][j] >= thr[rr]) ? (1u << (8 * rr + j)) : 0u;
        if (FILTER_ABLATION == FILTER_NO_EMIT) { sink |= mine; return; }
        mine |= __shfl_xor_sync(0xffffffffu, mine, 1);
        mine |= __shfl_xor_sync(0xffffffffu, mine, 2);
#pragma unroll
        for (int rr = 0; rr < 2; ++rr) {
          const int s = 2 * rr + H;   // compile-time: cnt[] stays in registers
          unsigned int m8 = (mine >> (8 * rr)) & 0xFFu;
#pragma unroll
          for (int t = 0; t < 8; ++t) {   // the set octets of this row in ascending order (quad-uniform trip count)
            if (!m8) break;
            const int j = __ffs(m8) - 1;
            m8 &= m8 - 1u;
            // the lane's score pair of octet j, selected by the bits of j (a runtime index would put acc in local memory)
            float a[8], b[8];
#pragma unroll
            for (int u = 0; u < 8; ++u) { a[u] = acc[4 * u + 2 * rr]; b[u] = acc[4 * u + 2 * rr + 1]; }
#pragma unroll
            for (int u = 0; u < 4; ++u) { a[u] = (j & 1) ? a[2 * u + 1] : a[2 * u]; b[u] = (j & 1) ? b[2 * u + 1] : b[2 * u]; }
#pragma unroll
            for (int u = 0; u < 2; ++u) { a[u] = (j & 2) ? a[2 * u + 1] : a[2 * u]; b[u] = (j & 2) ? b[2 * u + 1] : b[2 * u]; }
            if (cnt[s] < cap) {
              const long long seg = seg_base[rr] + (H ? cap : 0u) + cnt[s];
              reinterpret_cast<float2*>(p.cand_s + seg * 8)[lane & 3] = make_float2((j & 4) ? a[1] : a[0], (j & 4) ? b[1] : b[0]);
              if (quad_leader) p.cand_i[seg] = (unsigned int)(col0 + 64 * H + 8 * j);
              ++cnt[s];
            } else {
              ovf |= 1u << s;
            }
          }
        }
      }
    }
  };

  float acc0[32], acc1[32];   // column halves 0 / 1 of the current tile
  int stage = 0; uint32_t phase = 0;
  int prev_stage = 0; uint32_t prev_phase = 0;   // ring slot (and its fill parity) of the previous tile
  // One tile; half 0 of it is in acc0 and complete on entry.  Each epilogue runs while the MMAs of the next half are in
  // flight.  Nothing is in flight across the loop's back edge and the last tile is a separate instantiation: ptxas
  // serializes the wgmma when an accumulator is in flight at a loop head or only on some paths.
  auto tile_step = [&](int it, auto last_tile) {
    constexpr bool LAST = decltype(last_tile)::value;
    const long long col0 = (long long)(u_begin + it) * stride * TILE_N;  // zero-padded rows of the last tile score 0: dropped in finalize (idx >= N)
    issue(acc1, stage, 1);
    epilogue(acc0, col0, it, std::integral_constant<int, 0>{});
    const int next_stage = stage + 1 == STAGES ? 0 : stage + 1;
    const uint32_t next_phase = stage + 1 == STAGES ? phase ^ 1 : phase;
    if (!LAST) {
      mbar_wait(&full[next_stage], next_phase);
      issue(acc0, next_stage, 0);
      wgmma_wait<1>();          // half 1 has retired, half 0 of the next tile is in flight
    } else {
      wgmma_wait<0>();
    }
    acc_fence(acc1);
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty[stage]);   // both halves' MMAs on this slot have retired: it may be refilled
    // Refill one tile behind: the previous tile's slot, which the other warpgroups have had a whole tile's time to
    // release, so the issuer rarely waits on the slowest warpgroup.
    if (!LAST && issuer && it >= 1 && it - 1 + STAGES < n_iter) {
      mbar_wait(&empty[prev_stage], prev_phase);
      load_tile(it - 1 + STAGES, prev_stage);
    }
    prev_stage = stage; prev_phase = phase;
    stage = next_stage; phase = next_phase;
    epilogue(acc1, col0, it, std::integral_constant<int, 1>{});
    if (!LAST) {
      wgmma_wait<0>();
      acc_fence(acc0);
    }
  };
  if (n_iter > 0) {
    mbar_wait(&full[0], 0);
    issue(acc0, 0, 0);
    wgmma_wait<0>();
    acc_fence(acc0);
    for (int it = 0; it + 1 < n_iter; ++it) tile_step(it, std::false_type{});
    tile_step(n_iter - 1, std::true_type{});
  }
  if (MODE == MODE_SAMPLE) {
#pragma unroll
    for (int s = 0; s < 4; ++s) {   // bins this part did not fill
      const long long row = row_a + 8 * (s >> 1);
      if (quad_leader && row < p.Q)
        for (int b = bin_out; b < bins_per_part; ++b)
          p.binmax[row * p.bins_ld + (long long)part * bins_per_part * 2 + (s & 1) + 2 * b] = -INFINITY;
    }
  } else if (quad_leader) {
#pragma unroll
    for (int s = 0; s < 4; ++s)
      if (rescanned(row_a + 8 * (s >> 1)))
        p.count[((row_a + 8 * (s >> 1)) * p.parts + part) * 2 + (s & 1)] =
            FILTER_ABLATION != FILTER_FULL ? sink : ((ovf >> s) & 1u) ? (cap + 1u) : cnt[s];
  }
}

template <int KB, int STAGES, int MODE>
__global__ void __launch_bounds__(THREADS, 1)
tc_scan_kernel(const __grid_constant__ ScanParams p) {
  if constexpr (MODE == MODE_SAMPLE) {
    if (p.simg != nullptr && p.hdr->sample == SAMPLE_NORM) { tc_scan_body<KB, STAGES, MODE, true>(p); return; }
  }
  tc_scan_body<KB, STAGES, MODE, false>(p);
}

// ------------------------------------------------------------------------------------------------
// threshold from the bin maxima; finalize; fallback
// ------------------------------------------------------------------------------------------------
// orderable key: larger float <=> larger unsigned (NaN sorts above +inf; -0 < +0, callers canonicalise zeros)
__device__ __forceinline__ unsigned int f2key(float f) {
  unsigned int u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float key2f(unsigned int k) {
  return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}
// Rank key of an exactly scored candidate (local index < 2^31):
//   key(score, -0 folded onto +0) << 32 | (2^31 - 1 - index) << 1 | (score is -0.0f)
// The 64-bit order is (score desc, index asc), with -0 tied to +0 as in the exact path.  The low bit never decides an
// order (indices are unique); it carries the sign of a zero score, so the output keeps the chain's own bits.
__device__ __forceinline__ unsigned long long rank_key(float s, unsigned int idx) {
  const unsigned int lo = (0xFFFFFFFEu - 2u * idx) | (__float_as_uint(s) == 0x80000000u ? 1u : 0u);
  return ((unsigned long long)f2key(s + 0.0f) << 32) | lo;
}
__device__ __forceinline__ float rank_key_score(unsigned long long e) {   // the low bit is only ever set on a zero key
  return __uint_as_float(__float_as_uint(key2f((unsigned int)(e >> 32))) | ((unsigned int)e << 31));
}
__device__ __forceinline__ unsigned int rank_key_index(unsigned long long e) { return 0x7FFFFFFFu - ((unsigned int)e >> 1); }
__device__ __forceinline__ int warp_incl_scan(int v, int lane) {
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_up_sync(0xffffffffu, v, o); if (lane >= o) v += t; }
  return v;
}

// k-th largest of the keys a warp holds in registers (KPL per lane, unused slots = 0 = below every float key):
// bitwise binary search for the largest v with #{key >= v} >= k, one REDUX.SUM per bit.
template <int KPL>
__device__ __forceinline__ unsigned int warp_kth_largest_regs(const unsigned int (&key)[KPL], int k, unsigned int prefix = 0, int top_bit = 31) {
  // `prefix` = the bits above top_bit, known to be shared by every real key (unused slots are 0 and never reach it)
  for (int bit = top_bit; bit >= 0; --bit) {
    const unsigned int cand = prefix | (1u << bit);
    int c = 0;
#pragma unroll
    for (int j = 0; j < KPL; ++j) c += (key[j] >= cand) ? 1 : 0;
    c = __reduce_add_sync(0xffffffffu, c);
    if (c >= k) prefix = cand;
  }
  return prefix;
}
// the same over n keys in shared memory
__device__ __forceinline__ unsigned int warp_kth_largest_smem(const unsigned int* keys, int n, int k, int lane, unsigned int prefix, int top_bit) {
  for (int bit = top_bit; bit >= 0; --bit) {
    const unsigned int cand = prefix | (1u << bit);
    int c = 0;
    for (int t = lane; t < n; t += 32) c += (keys[t] >= cand) ? 1 : 0;
    c = __reduce_add_sync(0xffffffffu, c);
    if (c >= k) prefix = cand;
  }
  return prefix;
}

// (1b) K-th largest bin maximum of the sampled pass -> guaranteed threshold thr_safe = L_K - margin, and the filter
// threshold thr = L_K' - margin at the smaller bin rank k_filter (Plan::k_filter; == k where the threshold must stay a
// guarantee).  One warp per query, the query's <= 32*KPL bin maxima live in registers.
template <int KPL>
__device__ __forceinline__ void thresholds_of_row(const float* __restrict__ binmax, int bins_ld, int n_bins, int k, int k_filter,
                                                  const float* __restrict__ margin, float* __restrict__ thr, float* __restrict__ thr_safe,
                                                  unsigned int* __restrict__ overflow, unsigned int* __restrict__ retry, long long row, int lane) {
  const float* src = binmax + row * bins_ld;
  unsigned int key[KPL];
#pragma unroll
  for (int j = 0; j < KPL; ++j) { const int i = j * 32 + lane; key[j] = i < n_bins ? f2key(__ldg(src + i)) : 0u; }
  const float safe = key2f(warp_kth_largest_regs<KPL>(key, k)) - margin[row];
  const float filter = k_filter < k ? key2f(warp_kth_largest_regs<KPL>(key, k_filter)) - margin[row] : safe;
  if (lane == 0) { thr[row] = filter; thr_safe[row] = safe; overflow[row] = 0; retry[row] = 0; }
}
// On a norm-sample index
// (n_bins_norm > 0 and the header says so) the pass filled n_bins_norm bins and both thresholds sit at rank k.
template <int KPL>
__global__ void __launch_bounds__(256)
tc_threshold_kernel(const float* __restrict__ binmax, int bins_ld, int n_bins, int k, int k_filter, const float* __restrict__ margin,
                    float* __restrict__ thr, float* __restrict__ thr_safe, unsigned int* __restrict__ overflow,
                    unsigned int* __restrict__ retry, long long Q, const IndexHeader* __restrict__ hdr, int n_bins_norm) {
  const int lane = threadIdx.x & 31;
  const long long row = ((long long)blockIdx.x * 256 + threadIdx.x) >> 5;
  if (row >= Q) return;
  if (n_bins_norm > 0 && hdr->sample == SAMPLE_NORM) { n_bins = n_bins_norm; k_filter = k; }
  if (KPL > 16 && n_bins <= 512) thresholds_of_row<16>(binmax, bins_ld, n_bins, k, k_filter, margin, thr, thr_safe, overflow, retry, row, lane);
  else thresholds_of_row<KPL>(binmax, bins_ld, n_bins, k, k_filter, margin, thr, thr_safe, overflow, retry, row, lane);
}

// (3) finalize: one WARP per query, no block-wide barriers.
enum { FIN_TOPK = 0, FIN_EXCLUDE = 1, FIN_COUNT = 2 };
constexpr int FW_WARPS = 4;                       // queries per CTA of the fallback re-rank kernel
// Capacities per query come from the plan (they grow with k); a row that overflows them takes the exact fallback.
// overflow[row]: 0 = done, 1 = exact fallback
// retry[row]:    1 = the row's filter threshold was above thr_safe and missed; it was filtered again at thr_safe

struct FinParams {
  const float* q; const float* corpus; int d; int k; long long index_offset; long long N; long long Q;
  const unsigned int* count; const float* cand_s; const unsigned int* cand_i; int segs; int cap_part;
  const float* cut; float* thr; const float* thr_safe; unsigned int* overflow;
  unsigned int* retry; int retry_pass;           // retry_pass: the select launch after the retry filter pass (marked rows only)
  int cap_keys, cap_band;                        // survivors per query (keys in shared memory) / band entries re-scored exactly
  unsigned int* band_idx; int* band_n;           // [Qp, cap_band] local indices of the band, [Qp] their number
  int allow_short;                               // sharded scan with a GLOBAL threshold: a shard may hold fewer than k survivors
  float* out_s; long long* out_i;                // TOPK: [Q, k];  EXCLUDE: [Q, k_out]
  // EXCLUDE (k = k_out + n_excl candidates are fetched, then re-ranked)
  const long long* identifiers; const long long* exclusions; int n_excl; int k_out;
  // COUNT
  const float* pos; const int* qexp; const IndexHeader* hdr; int* out_count;
};

// exact score: the canonical sequential fmaf chain on the fp32 corpus row (bit-identical to the oracle)
__device__ __forceinline__ float exact_score(const float* __restrict__ qs, const float* __restrict__ c, int d) {
  float acc = 0.f;
  if ((d & 31) == 0) {  // 8 loads (128 B) in flight per step, then the canonical chain on them
    for (int kk = 0; kk < d; kk += 32) {
      float4 cv[8];
#pragma unroll
      for (int u = 0; u < 8; ++u) cv[u] = __ldg(reinterpret_cast<const float4*>(c + kk) + u);
#pragma unroll
      for (int u = 0; u < 8; ++u) {
        acc = fmaf(qs[kk + 4 * u], cv[u].x, acc); acc = fmaf(qs[kk + 4 * u + 1], cv[u].y, acc);
        acc = fmaf(qs[kk + 4 * u + 2], cv[u].z, acc); acc = fmaf(qs[kk + 4 * u + 3], cv[u].w, acc);
      }
    }
  } else if ((d & 3) == 0) {
    for (int kk = 0; kk < d; kk += 4) {
      const float4 cv = __ldg(reinterpret_cast<const float4*>(c + kk));
      acc = fmaf(qs[kk], cv.x, acc); acc = fmaf(qs[kk + 1], cv.y, acc);
      acc = fmaf(qs[kk + 2], cv.z, acc); acc = fmaf(qs[kk + 3], cv.w, acc);
    }
  } else {
    for (int kk = 0; kk < d; ++kk) acc = fmaf(qs[kk], __ldg(c + kk), acc);
  }
  return acc;  // the chain's own bits, -0.0f included (rank_key folds -0 onto +0 for the order)
}

// two independent chains at once (same arithmetic per chain as exact_score)
__device__ __forceinline__ void exact_score2(const float* __restrict__ qs, const float* __restrict__ c0, const float* __restrict__ c1,
                                             int d, float& s0, float& s1) {
  if ((d & 31) == 0) {
    float a0 = 0.f, a1 = 0.f;
    for (int kk = 0; kk < d; kk += 32) {
      float4 u0[8], u1[8];
#pragma unroll
      for (int u = 0; u < 8; ++u) { u0[u] = __ldg(reinterpret_cast<const float4*>(c0 + kk) + u); u1[u] = __ldg(reinterpret_cast<const float4*>(c1 + kk) + u); }
#pragma unroll
      for (int u = 0; u < 8; ++u) {
        const float q0 = qs[kk + 4 * u], q1 = qs[kk + 4 * u + 1], q2 = qs[kk + 4 * u + 2], q3 = qs[kk + 4 * u + 3];
        a0 = fmaf(q0, u0[u].x, a0); a1 = fmaf(q0, u1[u].x, a1);
        a0 = fmaf(q1, u0[u].y, a0); a1 = fmaf(q1, u1[u].y, a1);
        a0 = fmaf(q2, u0[u].z, a0); a1 = fmaf(q2, u1[u].z, a1);
        a0 = fmaf(q3, u0[u].w, a0); a1 = fmaf(q3, u1[u].w, a1);
      }
    }
    s0 = a0; s1 = a1;
  } else {
    s0 = exact_score(qs, c0, d); s1 = exact_score(qs, c1, d);
  }
}

// _exclude (layers/factorized_top_k.py:83-115) on a query's kf best candidates, sorted in `srt` as rank_key(score,
// local index): identifiers in `exclusions[row]` get score - 1e5, the k_out best ADJUSTED scores win (ties -> lower
// position), the ORIGINAL scores and indices are written.  One warp; akey = kf words of scratch.
__device__ __forceinline__ void exclude_rerank(const unsigned long long* srt, int kf, unsigned long long* akey, long long row,
                                               const FinParams& p, int lane) {
  for (int t = lane; t < kf; t += 32) {
    const unsigned long long e = srt[t];
    const float s = key2f((unsigned int)(e >> 32));
    const long long gi = (long long)rank_key_index(e) + p.index_offset;
    const long long ident = p.identifiers ? __ldg(p.identifiers + gi) : gi;
    bool isin = false;
    for (int x = 0; x < p.n_excl; ++x) isin |= (__ldg(p.exclusions + row * p.n_excl + x) == ident);
    const float adj = (isin ? s - 1.0e5f : s) + 0.0f;   // scores - isin * 1e5 (:104-107)
    akey[t] = ((unsigned long long)f2key(adj) << 32) | (unsigned long long)(0xFFFFFFFFu - (unsigned int)t);
  }
  __syncwarp();
  for (int t = lane; t < kf; t += 32) {
    const unsigned long long mine = akey[t];
    int rank = 0;
    for (int j = 0; j < kf; ++j) rank += (akey[j] > mine) ? 1 : 0;
    if (rank < p.k_out) {
      const unsigned long long e = srt[t];
      p.out_s[row * p.k_out + rank] = rank_key_score(e);
      p.out_i[row * p.k_out + rank] = (long long)rank_key_index(e) + p.index_offset;
    }
  }
}

// (3a) SELECT, one warp per query, no block-wide barriers, 4 KB of shared memory per query so that ~50 queries are
// in flight per SM (the work is a chain of dependent L2 round trips: occupancy is what hides it):
//   pass 1  survivors of the octet records -> their screening keys in shared memory;  tau = k-th largest (bitwise
//           search on register-resident keys);  lim = tau - 2 eps
//   pass 2  the records again: indices of the survivors with key >= lim  -> band_idx[row, :], band_n[row]
// COUNT mode needs one pass: #{screen > pos + eps} is counted, the indices with |screen - pos| <= eps form the band.
__host__ __device__ inline size_t sel_warp_bytes(int cap_keys, int segs) {
  return (size_t)cap_keys * 4 + (size_t)cap_keys * 2 + (size_t)((segs + 1 + 3) & ~3) * 4;
}
constexpr int SEL_WARPS = 8;

// one 32-record window of a query's octet records: lane -> (first index, 8 scores); returns false past the end
__device__ __forceinline__ bool load_record(const FinParams& p, long long row, const int* soff, int rec, int total_rec,
                                            unsigned int& ix0, float (&sc)[8]) {
  if (rec >= total_rec) return false;
  int lo = 0, hi = p.segs;  // largest segment with soff[seg] <= rec
  while (hi - lo > 1) { const int mid = (lo + hi) >> 1; if (soff[mid] <= rec) lo = mid; else hi = mid; }
  const long long at = (row * p.segs + lo) * p.cap_part + (rec - soff[lo]);
  ix0 = __ldg(p.cand_i + at);
  const float4 s0 = __ldg(reinterpret_cast<const float4*>(p.cand_s + at * 8));
  const float4 s1 = __ldg(reinterpret_cast<const float4*>(p.cand_s + at * 8) + 1);
  sc[0] = s0.x; sc[1] = s0.y; sc[2] = s0.z; sc[3] = s0.w; sc[4] = s1.x; sc[5] = s1.y; sc[6] = s1.z; sc[7] = s1.w;
  return true;
}

template <int MODE>
__global__ void __launch_bounds__(SEL_WARPS * 32)
tc_select_kernel(const FinParams p) {
  extern __shared__ __align__(16) unsigned char fsm[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long row = (long long)blockIdx.x * SEL_WARPS + warp;
  if (row >= p.Q || (p.retry_pass && p.retry[row] == 0u)) return;
  unsigned char* base = fsm + (size_t)warp * sel_warp_bytes(p.cap_keys, p.segs);
  unsigned int* keys = reinterpret_cast<unsigned int*>(base);                 // [cap_keys] screening keys
  unsigned short* loc = reinterpret_cast<unsigned short*>(keys + p.cap_keys);  // [cap_keys] (flat record index << 3 | column): total records < 8192
  int* soff = reinterpret_cast<int*>(loc + p.cap_keys);                        // [segs + 1]
  const unsigned int n32 = (unsigned int)p.N;   // N < 2^31
  unsigned int* band = p.band_idx + row * p.cap_band;

  // segment counts -> exclusive prefix
  int carry = 0; bool bad = false;
  for (int s0 = 0; s0 < p.segs; s0 += 32) {
    const int s = s0 + lane;
    int c = 0;
    if (s < p.segs) {
      const unsigned int cc = __ldg(p.count + row * p.segs + s);
      if (cc > (unsigned int)p.cap_part) bad = true; else c = (int)cc;
    }
    const int inc = warp_incl_scan(c, lane);
    if (s < p.segs) soff[s + 1] = carry + inc;
    carry += __shfl_sync(0xffffffffu, inc, 31);
  }
  if (lane == 0) soff[0] = 0;
  if (__any_sync(0xffffffffu, bad)) {  // a segment overflowed in the filter pass: records are missing -> exact fallback
    if (lane == 0) { p.overflow[row] = 1; p.band_n[row] = 0; }
    return;
  }
  __syncwarp();
  const int total_rec = soff[p.segs];
  const float thr_row = p.thr[row];
  if (MODE != FIN_COUNT && total_rec >= 8192) {   // the 16-bit record locator holds 13 bits of record index
    if (lane == 0) { p.overflow[row] = 1; p.band_n[row] = 0; }
    return;
  }

  if (MODE == FIN_COUNT) {
    // metrics/factorized_top_k.py:181-192: in_top_k(target = the positive, k) <=> #{candidates scoring > positive} < k.
    // screen > pos + eps => exact > pos (counted as is); |screen - pos| <= eps => re-scored exactly (3b).  When the
    // positive lies below the listed range, at least K listed candidates are definite (L_q > pos + eps), so
    // min(k, count) is exact.
    const float eps = 0.5f * p.cut[row];
    const float pos_s = ldexpf(p.pos[row], p.hdr->st.exp + p.qexp[row]);
    const float hi = pos_s + eps, lo_b = pos_s - eps;
    int definite = 0, m = 0;
    for (int rb = 0; rb < total_rec; rb += 32) {
      unsigned int ix0 = 0, amb = 0; int cnt = 0; float sc[8];
      if (load_record(p, row, soff, rb + lane, total_rec, ix0, sc)) {
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const bool real = ix0 + j < n32;
          definite += (real && sc[j] > hi) ? 1 : 0;
          const bool a = real && sc[j] > lo_b && !(sc[j] > hi);
          amb |= a ? (1u << j) : 0u; cnt += a ? 1 : 0;
        }
      }
      const int incl = warp_incl_scan(cnt, lane);
      const int tot = __shfl_sync(0xffffffffu, incl, 31);
      if (m + tot <= p.cap_band) {
        int at_pos = m + incl - cnt;
#pragma unroll
        for (int j = 0; j < 8; ++j)
          if (amb & (1u << j)) { band[at_pos] = ix0 + j; ++at_pos; }
      }
      m += tot;
    }
    definite = __reduce_add_sync(0xffffffffu, definite);
    if (lane == 0) {
      if (definite >= p.k) { p.out_count[row] = p.k; p.band_n[row] = 0; p.overflow[row] = 0; }
      else if (m > p.cap_band) { p.overflow[row] = 1; p.band_n[row] = 0; }
      else { p.out_count[row] = definite; p.band_n[row] = m; p.overflow[row] = 0; }   // 3b adds the re-scored ones
    }
    return;
  }

  // ---- TOPK / EXCLUDE, pass 1: screening keys of the survivors (score >= filter threshold, real row)
  int n = 0;
  unsigned int kmax = 0u, kmin = 0xFFFFFFFFu;
  for (int rb = 0; rb < total_rec; rb += 32) {
    float sc[8]; unsigned int ix0 = 0, keep = 0; int cnt = 0;
    if (load_record(p, row, soff, rb + lane, total_rec, ix0, sc)) {
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const bool kp = sc[j] >= thr_row && ix0 + j < n32;
        keep |= kp ? (1u << j) : 0u; cnt += kp ? 1 : 0;
      }
    }
    const int incl = warp_incl_scan(cnt, lane);
    const int tot = __shfl_sync(0xffffffffu, incl, 31);
    if (n + tot <= p.cap_keys) {   // warp-uniform: the stores below need no per-entry bound check
      int at_pos = n + incl - cnt;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        if (keep & (1u << j)) {
          const unsigned int key = f2key(sc[j] + 0.0f);   // -0 -> +0: key order == float order
          kmax = max(kmax, key); kmin = min(kmin, key);
          keys[at_pos] = key;
          loc[at_pos] = (unsigned short)(((rb + lane) << 3) | j);
          ++at_pos;
        }
      }
    }
    n += tot;
  }
  // A row whose filter threshold (bin rank k_filter) was above the guaranteed one and fails a check that a lower
  // threshold can pass (n >= k, lim >= thr) is marked for the retry filter pass at thr_safe; any other miss, and any
  // miss at thr_safe, takes the exact fallback.  Overflows (segments, records, survivor keys) grow as the threshold
  // drops, so they go straight to the fallback.
  auto miss = [&]() {
    if (lane == 0) {
      const float safe = p.thr_safe[row];
      if (thr_row > safe) { p.retry[row] = 1; p.thr[row] = safe; } else p.overflow[row] = 1;
      p.band_n[row] = 0;
    }
  };
  if (n > p.cap_keys) { if (lane == 0) { p.overflow[row] = 1; p.band_n[row] = 0; } return; }
  if (n < p.k && !p.allow_short) { miss(); return; }
  __syncwarp();
  if (n < p.k) {
    // Sharded scan, threshold agreed across the shards (see comm.cu): this shard holds fewer than k candidates above it.
    // Every one of them is re-scored and emitted -- members of the global top-k are survivors on their shard by construction.
    const bool fits = n <= p.cap_band;
    for (int t = lane; t < n && fits; t += 32) {
      const unsigned int l = loc[t];
      const int rec = (int)(l >> 3);
      int lo = 0, hi = p.segs;
      while (hi - lo > 1) { const int mid = (lo + hi) >> 1; if (soff[mid] <= rec) lo = mid; else hi = mid; }
      band[t] = __ldg(p.cand_i + (row * p.segs + lo) * p.cap_part + (rec - soff[lo])) + (l & 7u);
    }
    if (lane == 0) { p.overflow[row] = fits ? 0u : 1u; p.band_n[row] = fits ? n : 0; }
    return;
  }
  // tau = k-th best screening score: bitwise search below the bits the largest and the smallest key share
  kmax = __reduce_max_sync(0xffffffffu, kmax); kmin = __reduce_min_sync(0xffffffffu, kmin);
  unsigned int tau_key;
  {
    const unsigned int diff = kmax ^ kmin;
    const int top = diff ? (31 - __clz(diff)) : -1;           // highest bit in which the survivors differ
    const unsigned int prefix0 = top >= 31 ? 0u : (top < 0 ? kmax : (kmax & ~((2u << top) - 1u)));   // top == -1: all keys equal
    if (n <= 512) {
      unsigned int kr[16];
#pragma unroll
      for (int j = 0; j < 16; ++j) { const int t = j * 32 + lane; kr[j] = t < n ? keys[t] : 0u; }
      tau_key = warp_kth_largest_regs<16>(kr, p.k, prefix0, top);
    } else if (n <= 1024) {
      unsigned int kr[32];
#pragma unroll
      for (int j = 0; j < 32; ++j) { const int t = j * 32 + lane; kr[j] = t < n ? keys[t] : 0u; }
      tau_key = warp_kth_largest_regs<32>(kr, p.k, prefix0, top);
    } else {
      tau_key = warp_kth_largest_smem(keys, n, p.k, lane, prefix0, top);
    }
  }
  const float lim = key2f(tau_key) - p.cut[row];
  // Self-check that makes the threshold choice a pure performance matter: the whole band [lim, inf) must
  // lie above the filter threshold, otherwise survivors could be missing -> exact fallback.
  // (with a threshold agreed across shards the local band may reach below it: what is missing there cannot be in the
  //  GLOBAL top-k, and the local list is only an input of the cross-shard merge)
  if (!p.allow_short && (!(lim >= thr_row) || !(lim > -INFINITY))) { miss(); return; }
  // pass 2: only the band members (key >= key(lim)) go back to their record for the corpus index
  const unsigned int lim_key = f2key(lim + 0.0f);
  const unsigned int lt_mask = (1u << lane) - 1u;
  int m = 0;
  for (int tb = 0; tb < n; tb += 32) {
    const int t = tb + lane;
    const bool kp = t < n && keys[t] >= lim_key;
    const unsigned int vote = __ballot_sync(0xffffffffu, kp);
    if (kp) {
      const int at_pos = m + __popc(vote & lt_mask);
      if (at_pos < p.cap_band) {
        const unsigned int l = loc[t];
        const int rec = (int)(l >> 3);
        int lo = 0, hi = p.segs;
        while (hi - lo > 1) { const int mid = (lo + hi) >> 1; if (soff[mid] <= rec) lo = mid; else hi = mid; }
        band[at_pos] = __ldg(p.cand_i + (row * p.segs + lo) * p.cap_part + (rec - soff[lo])) + (l & 7u);
      }
    }
    m += __popc(vote);
  }
  if (lane == 0) {
    if (m > p.cap_band) { p.overflow[row] = 1; p.band_n[row] = 0; }   // band too crowded (massive ties)
    else { p.overflow[row] = 0; p.band_n[row] = m; }
  }
}

// (3b) RE-SCORE + RANK, one 128-thread block per query: every band candidate's fp32 corpus row is fetched at once (one
// DRAM round trip per query; ~115 MB of random 256-byte rows per cfg2 batch, the HBM-bound part of the finalize step),
// the canonical fmaf chain gives the exact score, and each thread ranks its entry against the band in shared memory
// (ranks are unique: (score desc, index asc) is a total order).  EXCLUDE re-ranks the k best, COUNT adds #{exact > pos}.
constexpr int RS_BLOCK = 128;
template <int MODE>
__global__ void __launch_bounds__(RS_BLOCK)
tc_rescore_kernel(const FinParams p) {
  extern __shared__ __align__(16) unsigned char rsm[];
  unsigned long long* sk = reinterpret_cast<unsigned long long*>(rsm);                  // [cap_band] composite keys
  float* qs = reinterpret_cast<float*>(sk + p.cap_band);                                  // [d]
  unsigned long long* srt = reinterpret_cast<unsigned long long*>(qs + ((p.d + 3) & ~3)); // EXCLUDE: [2 * k]
  __shared__ int greater_sh;
  const long long row = blockIdx.x;
  const int tid = threadIdx.x;
  if (p.overflow[row] != 0) return;
  const int m = p.band_n[row];
  if (MODE == FIN_COUNT && m == 0) return;    // the select kernel already wrote the count
  for (int t = tid; t < p.d; t += RS_BLOCK) qs[t] = p.q[row * p.d + t];
  if (tid == 0) greater_sh = 0;
  __syncthreads();
  const unsigned int* band = p.band_idx + row * p.cap_band;
  if (MODE == FIN_COUNT) {
    const float pos = p.pos[row];
    int g = 0;
    for (int t = tid; t < m; t += RS_BLOCK) g += (exact_score(qs, p.corpus + (long long)band[t] * p.d, p.d) > pos) ? 1 : 0;
    g = __reduce_add_sync(0xffffffffu, g);
    if ((tid & 31) == 0 && g) atomicAdd(&greater_sh, g);
    __syncthreads();
    if (tid == 0) { const int c = p.out_count[row] + greater_sh; p.out_count[row] = c < p.k ? c : p.k; }
    return;
  }
  if (p.d == 64) {
    // d = 64 (the headline shape): EIGHT lanes fetch one 256-byte corpus row (32 bytes each, one coalesced request per row;
    // every row of the band is in flight before the first FMA), then the canonical chain k = 0..63 walks through the eight
    // lanes with the accumulator handed on by shuffle -- same arithmetic, same order, same bits as exact_score().
    constexpr int RPB = RS_BLOCK / 8;          // rows per block round
    constexpr int MAXR = 8;                    // rounds held in registers (m <= 128); larger bands loop
    const int sub = tid & 7, grp = tid >> 3;
    for (int t0 = 0; t0 < m; t0 += RPB * MAXR) {
      float4 a[MAXR], b[MAXR];
#pragma unroll
      for (int r = 0; r < MAXR; ++r) {
        const int t = t0 + r * RPB + grp;
        if (t < m) {
          const float4* src = reinterpret_cast<const float4*>(p.corpus + (long long)band[t] * 64) + sub * 2;
          a[r] = __ldg(src); b[r] = __ldg(src + 1);
        }
      }
      const float q0 = qs[sub * 8], q1 = qs[sub * 8 + 1], q2 = qs[sub * 8 + 2], q3 = qs[sub * 8 + 3];
      const float q4 = qs[sub * 8 + 4], q5 = qs[sub * 8 + 5], q6 = qs[sub * 8 + 6], q7 = qs[sub * 8 + 7];
#pragma unroll
      for (int r = 0; r < MAXR; ++r) {
        const int t = t0 + r * RPB + grp;
        const bool live = t < m;                    // uniform per 8-lane group; the shuffles below are executed by all lanes
        float acc = 0.f;
#pragma unroll
        for (int step = 0; step < 8; ++step) {
          if (sub == step && live) {
            acc = fmaf(q0, a[r].x, acc); acc = fmaf(q1, a[r].y, acc); acc = fmaf(q2, a[r].z, acc); acc = fmaf(q3, a[r].w, acc);
            acc = fmaf(q4, b[r].x, acc); acc = fmaf(q5, b[r].y, acc); acc = fmaf(q6, b[r].z, acc); acc = fmaf(q7, b[r].w, acc);
          }
          acc = __shfl_sync(0xffffffffu, acc, (threadIdx.x & 24) | step);   // hand the accumulator to the next lane of the group
        }
        if (live && sub == 0) sk[t] = rank_key(acc, band[t]);
      }
    }
  } else {
    for (int t = tid; t < m; t += RS_BLOCK) {
      const unsigned int idx = band[t];
      sk[t] = rank_key(exact_score(qs, p.corpus + (long long)idx * p.d, p.d), idx);
    }
  }
  __syncthreads();
  if (MODE == FIN_TOPK && m < p.k)   // short shard list: pad with (-inf, INT64_MAX), the merge's "no entry"
    for (int t = m + tid; t < p.k; t += RS_BLOCK) { p.out_s[row * p.k + t] = -INFINITY; p.out_i[row * p.k + t] = LLONG_MAX; }
  for (int t = tid; t < m; t += RS_BLOCK) {
    const unsigned long long mine = sk[t];
    int rank = 0;
#pragma unroll 4
    for (int j = 0; j < m; ++j) rank += (sk[j] > mine) ? 1 : 0;
    if (rank < p.k) {
      if (MODE == FIN_TOPK) {
        p.out_s[row * p.k + rank] = rank_key_score(mine);
        p.out_i[row * p.k + rank] = (long long)rank_key_index(mine) + p.index_offset;
      } else {
        srt[rank] = mine;
      }
    }
  }
  if (MODE == FIN_EXCLUDE) {
    __syncthreads();
    if (tid < 32) exclude_rerank(srt, p.k, srt + p.k, row, p, tid);
  }
}

// EXCLUDE for the rows the exact fallback produced: tmp_[s,i] [Q, k] sorted lists -> the same re-ranking
__global__ void __launch_bounds__(FW_WARPS * 32)
tc_exclude_fallback_kernel(const FinParams p, const float* __restrict__ tmp_s, const long long* __restrict__ tmp_i,
                           const unsigned int* __restrict__ was_fallback) {
  extern __shared__ __align__(16) unsigned char fsm[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long row = (long long)blockIdx.x * FW_WARPS + warp;
  if (row >= p.Q || was_fallback[row] == 0) return;
  unsigned long long* srt = reinterpret_cast<unsigned long long*>(fsm) + (size_t)warp * 2 * p.k;
  unsigned long long* akey = srt + p.k;
  for (int t = lane; t < p.k; t += 32)
    srt[t] = rank_key(tmp_s[row * p.k + t], (unsigned int)(tmp_i[row * p.k + t] - p.index_offset));
  __syncwarp();
  exclude_rerank(srt, p.k, akey, row, p, lane);
}

struct FallbackProvider {
  const float* q; const float* corpus; long long N; int d; long long index_offset; const unsigned int* overflow;
  float* qs;
  __device__ void begin(int row, void* extra) {
    qs = reinterpret_cast<float*>(extra);
    if (overflow[row] != 0) for (int t = threadIdx.x; t < d; t += blockDim.x) qs[t] = q[(long long)row * d + t];
  }
  __device__ long long count(int row) const { return overflow[row] != 0 ? N : 0; }
  __device__ void get(int, long long t, float& s, long long& i) const {
    const float* c = corpus + t * d;
    float acc = 0.f;
    for (int kk = 0; kk < d; ++kk) acc = fmaf(qs[kk], __ldg(c + kk), acc);
    s = acc; i = index_offset + t;   // the chain's own bits: row_topk_kernel compares floats (-0 == +0)
  }
};

// COUNT for the rows that overflowed: exact #{candidates scoring above the positive}, clipped at k
__global__ void __launch_bounds__(256)
tc_count_fallback_kernel(const float* __restrict__ q, const float* __restrict__ corpus, long long N, int d, int k,
                         const float* __restrict__ pos, const unsigned int* __restrict__ overflow, int* __restrict__ out_count) {
  __shared__ float qs[128];
  __shared__ int total;
  const int row = blockIdx.x;
  if (overflow[row] == 0) return;
  for (int t = threadIdx.x; t < d; t += 256) qs[t] = q[(long long)row * d + t];
  if (threadIdx.x == 0) total = 0;
  __syncthreads();
  const float ps = pos[row];
  int c = 0;
  for (long long t = threadIdx.x; t < N; t += 256) {
    const float* cr = corpus + t * d;
    float acc = 0.f;
    for (int kk = 0; kk < d; ++kk) acc = fmaf(qs[kk], __ldg(cr + kk), acc);
    c += (acc + 0.0f > ps) ? 1 : 0;
  }
  c = __reduce_add_sync(0xffffffffu, c);
  if ((threadIdx.x & 31) == 0) atomicAdd(&total, c);
  __syncthreads();
  if (threadIdx.x == 0) out_count[row] = total < k ? total : k;
}

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------
// Optional per-stage device timing (bench.py's roofline leg): CUDA events recorded on the launch stream
// around the stages of the call.  Off by default; adds two event records per stage when on.
struct Prof {
  bool on = false;
  static constexpr int MAXC = 512, STAGES_ = 4;  // 0 prep, 1 sample(+threshold), 2 filter, 3 finalize(+fallback)
  cudaEvent_t ev[MAXC][STAGES_ + 1];
  int created = 0, calls = 0;
};
static Prof g_prof;
static void prof_mark(cudaStream_t st, int stage) {
  if (!g_prof.on || g_prof.calls >= Prof::MAXC) return;
  int c = g_prof.calls;
  while (g_prof.created <= c) {
    for (int s = 0; s <= Prof::STAGES_; ++s) cudaEventCreate(&g_prof.ev[g_prof.created][s]);
    ++g_prof.created;
  }
  cudaEventRecord(g_prof.ev[c][stage], st);
  if (stage == Prof::STAGES_) ++g_prof.calls;
}

struct Plan {
  int kb, stages; long long n_tiles; int nqb; long long Qp;
  int stride, n_sample, group, bins_per_part, n_bins, bins_ld, parts_sample, parts_full, cap_part, cap_keys, cap_band;
  int k_filter;   // bin rank of the filter threshold of TOPK / EXCLUDE calls (filter_bin_rank)
  // the sampled pass on a norm-sample index: its tiles, and bins of `group_norm` tiles (0: the shape has no such index)
  int n_seq_norm, group_norm, bins_per_part_norm, n_bins_norm;
  size_t smem;
  // workspace offsets
  size_t o_qimg, o_margin, o_cut, o_thr, o_qexp, o_count, o_ovf, o_binmax, o_cand, o_tmp, o_band, o_bandn, o_thr_safe, o_retry,
      total;
};

// The bin rank K' of the filter threshold: the smallest rank with P(Binomial(k - 1, 1/stride) >= K') <= 1e-9, capped at k.
// L_K' (the K'-th largest bin maximum) is below tau, the k-th best screening score, unless K' of the k - 1 scores above
// tau sit in sampled tiles, one per bin; for a row in random order each of them does so with probability 1/stride.  A
// row that meets those odds anyway is caught by the select kernel's self-check and retried at L_k, which is always a
// lower bound (DESIGN.md, K2).
static int filter_bin_rank(int k, int stride) {
  if (stride <= 1 || k <= 1) return k;   // every tile is sampled: only rank k is a bound
  const int n = k - 1;
  const double p = 1.0 / stride;
  double tail = 0.0;   // P(X >= r), summed from the top
  for (int r = n; r >= 1; --r) {
    tail += exp(lgamma(n + 1.0) - lgamma(r + 1.0) - lgamma(n - r + 1.0) + r * log(p) + (n - r) * log1p(-p));
    if (tail > 1e-9) return r + 1;
  }
  return 1;
}

static bool make_plan(long long Q, long long N, int d, int k, Plan& pl) {
  if (d <= 0 || d > 128 || Q <= 0 || N <= 0 || k <= 0) return false;   // d > 128: smem budget (A blocks + ring) not laid out
  pl.kb = (d + KSLAB - 1) / KSLAB;
  pl.stages = pl.kb == 1 ? 6 : 4;
  pl.n_tiles = ceil_div(N, TILE_N);
  pl.nqb = (int)ceil_div(Q, QBLK);
  pl.Qp = (long long)pl.nqb * QBLK;
  if (k > 256 || N >= (1ll << 31)) return false;   // finalize capacities are sized for ~4k survivors + band entries per query
  // sample every stride-th tile; keep at least 4k raw (tile, half) bins so the k-th largest bin max is a tight bound
  const long long full_tiles = N / TILE_N;  // the zero-padded last tile is never sampled (its 0 scores are not candidates)
  if (full_tiles < 1) return false;
  pl.stride = MAX_SAMPLE_STRIDE;
#ifdef TFRS_DEBUG_SWITCHES
  { static int ov = getenv("TFRS_TC_SAMPLE_STRIDE") ? atoi(getenv("TFRS_TC_SAMPLE_STRIDE")) : 0; if (ov >= 1 && ov <= 16) pl.stride = ov; }
#endif
  while (pl.stride > 1 && 2 * ceil_div(full_tiles, pl.stride) < 4ll * k) pl.stride >>= 1;
  pl.k_filter = filter_bin_rank(k, pl.stride);
  pl.n_sample = (int)ceil_div(full_tiles, pl.stride);
  if (2ll * pl.n_sample < 4ll * k) return false;  // too few bins for a useful threshold -> caller uses the exact path
  const int sms = sm_count();
  int parts = sms / pl.nqb; if (parts < 1) parts = 1; if (parts > FIN_MAX_PARTS / 2) parts = FIN_MAX_PARTS / 2;
  pl.parts_sample = parts < pl.n_sample ? parts : pl.n_sample;
  pl.parts_full = (long long)parts < pl.n_tiles ? parts : (int)pl.n_tiles;
  {
    // one bin = `group` consecutive sampled tiles x 64 columns of an epilogue thread; <= max(512, 4k) <= MAX_BINS per query
    const int iters_max = (int)ceil_div(pl.n_sample, pl.parts_sample);
    const int target = 4 * k > 512 ? 4 * k : 512;
    int g = 1;
    while ((long long)pl.parts_sample * ceil_div(iters_max, g) * 2 > target && g < iters_max) ++g;
    pl.group = g;
    pl.bins_per_part = (int)ceil_div(iters_max, g);
    pl.n_bins = pl.parts_sample * pl.bins_per_part * 2;
    if (pl.n_bins > MAX_BINS || pl.n_bins < 2 * k) return false;
    // The norm sample runs on the same CTAs with groups of fewer tiles, up to MAX_BINS bins: its threshold is a
    // guarantee at rank k, and finer bins keep it tight.
    pl.n_seq_norm = (int)norm_sample_tiles(N);
    pl.group_norm = pl.bins_per_part_norm = pl.n_bins_norm = 0;
    if (pl.n_seq_norm >= pl.parts_sample) {
      const int iters_norm = (int)ceil_div(pl.n_seq_norm, pl.parts_sample);
      int gn = 1;
      while ((long long)pl.parts_sample * ceil_div(iters_norm, gn) * 2 > MAX_BINS) ++gn;
      const int bpp = (int)ceil_div(iters_norm, gn);
      if (pl.parts_sample * bpp * 2 >= 4 * k) { pl.group_norm = gn; pl.bins_per_part_norm = bpp; pl.n_bins_norm = pl.parts_sample * bpp * 2; }
    }
    if (pl.n_bins_norm == 0) pl.n_seq_norm = 0;
    const int bins_max = pl.n_bins > pl.n_bins_norm ? pl.n_bins : pl.n_bins_norm;
    pl.bins_ld = (bins_max + 31) / 32 * 32;
  }
  {
    // octet records per (part, column-half) segment: expected lambda = k * stride / segments (the threshold sits near rank
    // 1.2 k / sampled fraction, ~0.8 records per survivor); capacity = 2 lambda + 12 sqrt(lambda) + 8, a power of two in 32..512
    const double lambda = (double)k * pl.stride / (pl.parts_full * 2.0);
    const double want = 2.0 * lambda + 12.0 * sqrt(lambda) + 8.0;
    int p2 = 32; while (p2 < want && p2 < 512) p2 <<= 1;
    pl.cap_part = p2;
    // finalize capacities per query: ~1.3 k * stride survivors are expected (+60 %), the re-scored band holds ~k + the
    // candidates within 2 eps of tau
    int ck = 1024; while (ck < 1.6 * 1.3 * k * pl.stride && ck < 4096) ck <<= 1;
    pl.cap_keys = ck;                 // the re-scored band holds cap_keys / 2 >= 512 entries (~k + the candidates within 2 eps of tau)
    pl.cap_band = ck / 2;
  }
  pl.smem = (size_t)(2 + pl.stages) * pl.kb * SLAB_BYTES + 1024 /*align*/ + 256 /*barriers*/;
  size_t o = 0;
  auto take = [&](size_t bytes) { size_t r = o; o += align_up(bytes, 1024); return r; };
  pl.o_qimg = take((size_t)pl.nqb * 2 * pl.kb * SLAB_BYTES);
  pl.o_margin = take((size_t)pl.Qp * 4);
  pl.o_cut = take((size_t)pl.Qp * 4);
  pl.o_thr = take((size_t)pl.Qp * 4);
  pl.o_qexp = take((size_t)pl.Qp * 4);
  pl.o_count = take((size_t)pl.Qp * pl.parts_full * 2 * 4);
  pl.o_ovf = take((size_t)pl.Qp * 4);
  pl.o_binmax = take((size_t)pl.Qp * pl.bins_ld * 4);
  pl.o_cand = take((size_t)pl.Qp * pl.parts_full * 2 * pl.cap_part * (8 * 4 + 4));
  pl.o_tmp = take((size_t)Q * k * 12);   // EXCLUDE: the exact fallback's [Q, k] lists before the re-ranking
  pl.o_band = take((size_t)pl.Qp * pl.cap_band * 4);
  pl.o_bandn = take((size_t)pl.Qp * 4);
  pl.o_thr_safe = take((size_t)pl.Qp * 4);
  pl.o_retry = take((size_t)pl.Qp * 4);
  pl.total = o;
  return true;
}

template <int KB, int STAGES>
static int launch_scans(const Plan& pl, ScanParams sp, cudaStream_t st, int mode) {
  auto ks = tc_scan_kernel<KB, STAGES, MODE_SAMPLE>;
  auto kf = tc_scan_kernel<KB, STAGES, MODE_FILTER>;
  TFRS_DYN_SMEM(ks, (int)pl.smem);
  TFRS_DYN_SMEM(kf, (int)pl.smem);
  if (mode == MODE_SAMPLE) {
    sp.parts = pl.parts_sample; sp.n_seq = pl.n_sample; sp.stride = pl.stride;
    ks<<<(unsigned)(pl.nqb * sp.parts), THREADS, pl.smem, st>>>(sp);
  } else {
    sp.parts = pl.parts_full; sp.n_seq = (int)pl.n_tiles; sp.stride = 1;
    kf<<<(unsigned)(pl.nqb * sp.parts), THREADS, pl.smem, st>>>(sp);
  }
  TFRS_LAUNCH_CHECK();
  return TFRS_OK;
}

static int launch_scan_mode(const Plan& pl, const ScanParams& sp, cudaStream_t st, int mode) {
  if (pl.kb == 1) return launch_scans<1, 6>(pl, sp, st, mode);
  return launch_scans<2, 4>(pl, sp, st, mode);
}

// select; with `retry`, the filter pass and the select again for the rows the first select marked (launched
// unconditionally: no host sync; CTAs and warps without a marked row exit at once); then the exact re-scoring
template <int MODE>
static int launch_finalize(FinParams fp, const Plan& pl, ScanParams sp, bool retry, cudaStream_t st) {
  auto ksel = tc_select_kernel<MODE>;
  auto krs = tc_rescore_kernel<MODE>;
  TFRS_DYN_SMEM(ksel, (int)(SEL_WARPS * sel_warp_bytes(4096, FIN_MAX_PARTS)));
  ksel<<<(unsigned)ceil_div(fp.Q, SEL_WARPS), SEL_WARPS * 32, SEL_WARPS * sel_warp_bytes(fp.cap_keys, fp.segs), st>>>(fp);
  TFRS_LAUNCH_CHECK();
  if (retry) {
    sp.retry = fp.retry;
    const int rc = launch_scan_mode(pl, sp, st, MODE_FILTER);
    if (rc) return rc;
    fp.retry_pass = 1;
    ksel<<<(unsigned)ceil_div(fp.Q, SEL_WARPS), SEL_WARPS * 32, SEL_WARPS * sel_warp_bytes(fp.cap_keys, fp.segs), st>>>(fp);
    TFRS_LAUNCH_CHECK();
  }
  const size_t rs_smem = (size_t)fp.cap_band * 8 + (size_t)((fp.d + 3) & ~3) * 4 + (MODE == FIN_EXCLUDE ? (size_t)fp.k * 16 : 0);
  TFRS_DYN_SMEM(krs, 64 * 1024);
  krs<<<(unsigned)fp.Q, RS_BLOCK, rs_smem, st>>>(fp);
  TFRS_LAUNCH_CHECK();
  return TFRS_OK;
}

// One call = qprep -> sampled pass -> threshold -> filter pass -> finalize (+ retry, + exact fallback).
struct Call {
  int mode;  // FIN_*
  const float* q; long long Q; const float* corpus; const void* index_buf; long long N; int d; int k; long long index_offset;
  void* ws; size_t ws_bytes; cudaStream_t st;
  float* out_s; long long* out_i;                                                       // TOPK / EXCLUDE
  const long long* identifiers; const long long* exclusions; int n_excl; int k_out;     // EXCLUDE
  const float* pos; int* out_count;                                                     // COUNT
  // sharded scan: called between the threshold kernel and the filter pass with the device arrays that define the filter
  // thresholds; may raise thr[] (comm.cu exchanges a global lower bound of the k-th best score across the shards)
  ThrHook hook; void* hook_ctx; int allow_short;
};

static int run_call(const Call& c) {
  Plan pl;
  if (!make_plan(c.Q, c.N, c.d, c.k, pl)) {
    set_error("topk_tc: shape (Q=%lld N=%lld d=%d k=%d) is outside the tensor-core path; use tfrs_topk_scan_f32",
              c.Q, c.N, c.d, c.k);
    return TFRS_ERR_UNSUPPORTED;
  }
  if (!c.ws || c.ws_bytes < pl.total + 16) { set_error("topk_tc: workspace too small (%zu < %zu)", c.ws_bytes, pl.total + 16); return TFRS_ERR_WORKSPACE_TOO_SMALL; }
  // the exact re-scoring (exact_score, the d = 64 band loader) reads fp32 corpus rows as float4 when d % 4 == 0
  TFRS_CHECK_ARG((c.d & 3) != 0 || (reinterpret_cast<uintptr_t>(c.corpus) & 15) == 0,
                 "topk_tc: the corpus must be 16-byte aligned when d %% 4 == 0 (d=%d); pass an aligned copy", c.d);
  cudaStream_t st = c.st;
  unsigned char* w = (unsigned char*)(((uintptr_t)c.ws + 15) & ~(uintptr_t)15);
  unsigned char* qimg = w + pl.o_qimg;
  float* margin = (float*)(w + pl.o_margin);
  float* cut = (float*)(w + pl.o_cut);
  float* thr = (float*)(w + pl.o_thr);
  int* qexp = (int*)(w + pl.o_qexp);
  unsigned int* count = (unsigned int*)(w + pl.o_count);
  unsigned int* ovf = (unsigned int*)(w + pl.o_ovf);
  float* binmax = (float*)(w + pl.o_binmax);
  float* cand_s = (float*)(w + pl.o_cand);
  unsigned int* cand_i = (unsigned int*)(w + pl.o_cand + (size_t)pl.Qp * pl.parts_full * 2 * pl.cap_part * 32);
  float* tmp_s = (float*)(w + pl.o_tmp);
  long long* tmp_i = (long long*)(w + pl.o_tmp + align_up((size_t)c.Q * c.k * 4, 8));
  float* thr_safe = (float*)(w + pl.o_thr_safe);
  unsigned int* retry = (unsigned int*)(w + pl.o_retry);
  const IndexHeader* hdr = (const IndexHeader*)c.index_buf;
  const unsigned char* cimg = (const unsigned char*)c.index_buf + HEADER_BYTES;
  // The raised filter threshold needs the select kernel's self-check behind it: COUNT has none (its count of definite
  // candidates leans on L_k itself) and a sharded call turns it off (allow_short), so both keep the guaranteed bound.
  const int k_filter = (c.mode == FIN_COUNT || c.hook) ? c.k : pl.k_filter;

  prof_mark(st, 0);
  // (0) per-row exponent, image and margins: one launch
  tc_qprep_kernel<<<(unsigned)ceil_div(pl.Qp * 32, 256), 256, 0, st>>>(c.q, c.Q, pl.Qp, c.d, pl.kb, hdr, qimg, margin, cut, qexp);
  TFRS_LAUNCH_CHECK();
  ScanParams sp{};
  sp.qimg = qimg; sp.cimg = cimg; sp.Q = c.Q; sp.N = c.N; sp.nqb = pl.nqb; sp.n_tiles = pl.n_tiles;
  sp.binmax = binmax; sp.bins_ld = pl.bins_ld; sp.group = pl.group; sp.bins_per_part = pl.bins_per_part;
  sp.hdr = hdr;
  sp.simg = pl.n_bins_norm > 0 ? cimg + pl.n_tiles * pl.kb * (long long)SLAB_BYTES : nullptr;
  sp.n_seq_norm = pl.n_seq_norm; sp.group_norm = pl.group_norm; sp.bins_per_part_norm = pl.bins_per_part_norm;
  sp.thr = thr; sp.count = count; sp.cand_s = cand_s; sp.cand_i = cand_i; sp.cap_part = pl.cap_part;
  prof_mark(st, 1);
  // (1) sampled pass -> bin maxima -> k-th largest -> threshold
  int rc = launch_scan_mode(pl, sp, st, MODE_SAMPLE);
  if (rc) return rc;
  if (pl.n_bins <= 512 && pl.n_bins_norm <= 512)
    tc_threshold_kernel<16><<<(unsigned)ceil_div(c.Q * 32, 256), 256, 0, st>>>(binmax, pl.bins_ld, pl.n_bins, c.k, k_filter, margin,
                                                                                 thr, thr_safe, ovf, retry, c.Q, hdr, pl.n_bins_norm);
  else
    tc_threshold_kernel<32><<<(unsigned)ceil_div(c.Q * 32, 256), 256, 0, st>>>(binmax, pl.bins_ld, pl.n_bins, c.k, k_filter, margin,
                                                                                 thr, thr_safe, ovf, retry, c.Q, hdr, pl.n_bins_norm);
  TFRS_LAUNCH_CHECK();
  if (c.hook) {
    rc = c.hook(c.hook_ctx, thr, margin, cut, qexp, &hdr->st.exp, c.Q, st);
    if (rc) return rc;
  }
  prof_mark(st, 2);
  // (2) full pass with the fused threshold filter
  rc = launch_scan_mode(pl, sp, st, MODE_FILTER);
  if (rc) return rc;
  prof_mark(st, 3);
  if (FILTER_ABLATION != FILTER_FULL) { prof_mark(st, 4); return TFRS_OK; }   // no records: the outputs are not written
  // (3) exact re-scoring + final order (a warp per query); (4) exact fallback for the rows that asked for it
  FinParams fp{};
  fp.q = c.q; fp.corpus = c.corpus; fp.d = c.d; fp.k = c.k; fp.index_offset = c.index_offset; fp.N = c.N; fp.Q = c.Q;
  fp.count = count; fp.cand_s = cand_s; fp.cand_i = cand_i; fp.segs = pl.parts_full * 2; fp.cap_part = pl.cap_part;
  fp.cut = cut; fp.thr = thr; fp.thr_safe = thr_safe; fp.overflow = ovf; fp.retry = retry; fp.out_s = c.out_s; fp.out_i = c.out_i;
  fp.cap_keys = pl.cap_keys; fp.cap_band = pl.cap_band; fp.allow_short = c.allow_short;
  fp.band_idx = (unsigned int*)(w + pl.o_band); fp.band_n = (int*)(w + pl.o_bandn);
  fp.identifiers = c.identifiers; fp.exclusions = c.exclusions; fp.n_excl = c.n_excl; fp.k_out = c.k_out;
  fp.pos = c.pos; fp.qexp = qexp; fp.hdr = hdr; fp.out_count = c.out_count;
  const bool may_retry = k_filter < c.k;
  if (c.mode == FIN_TOPK) rc = launch_finalize<FIN_TOPK>(fp, pl, sp, may_retry, st);
  else if (c.mode == FIN_EXCLUDE) rc = launch_finalize<FIN_EXCLUDE>(fp, pl, sp, may_retry, st);
  else rc = launch_finalize<FIN_COUNT>(fp, pl, sp, false, st);
  if (rc) return rc;
  if (c.mode == FIN_COUNT) {
    tc_count_fallback_kernel<<<(unsigned)c.Q, 256, 0, st>>>(c.q, c.corpus, c.N, c.d, c.k, c.pos, ovf, c.out_count);
    TFRS_LAUNCH_CHECK();
  } else {
    // CTAs of non-flagged queries exit immediately
    FallbackProvider prov{c.q, c.corpus, c.N, c.d, c.index_offset, ovf, nullptr};
    int cap = rowselect_cap(c.k);
    TFRS_DYN_SMEM(row_topk_kernel<FallbackProvider>, 64 * 1024);
    float* fs = c.mode == FIN_TOPK ? c.out_s : tmp_s;
    long long* fi = c.mode == FIN_TOPK ? c.out_i : tmp_i;
    row_topk_kernel<FallbackProvider><<<(unsigned)c.Q, RS_THREADS, rowselect_smem(cap, (size_t)c.d * 4), st>>>(prov, c.k, cap, fs, fi, c.k);
    TFRS_LAUNCH_CHECK();
    if (c.mode == FIN_EXCLUDE) {
      tc_exclude_fallback_kernel<<<(unsigned)ceil_div(c.Q, FW_WARPS), FW_WARPS * 32, (size_t)FW_WARPS * 2 * c.k * 8, st>>>(fp, tmp_s, tmp_i, ovf);
      TFRS_LAUNCH_CHECK();
    }
  }
  prof_mark(st, 4);
  return TFRS_OK;
}

}  // namespace tc
}  // namespace tfrs

using namespace tfrs;
using namespace tfrs::tc;

extern "C" size_t tfrs_index_bytes(int64_t N, int d) {
  if (N <= 0 || d <= 0 || d > 128) return 0;
  int kb = (d + KSLAB - 1) / KSLAB;
  // [header][corpus image][norm-sample image, from 2^19 rows: N/8 rows more]
  return (size_t)HEADER_BYTES + (size_t)(ceil_div(N, TILE_N) + norm_sample_tiles(N)) * kb * SLAB_BYTES;
}

extern "C" int tfrs_index_build(const float* corpus, int64_t N, int d, void* index_buf, size_t index_bytes, void* stream) {
  TFRS_CHECK_ARG(corpus && index_buf && N > 0 && d > 0, "index_build: bad arguments");
  if (d > 128) { set_error("index_build: d=%d > 128 is not supported by the tensor-core path", d); return TFRS_ERR_UNSUPPORTED; }
  TFRS_CHECK_ARG(index_bytes >= tfrs_index_bytes(N, d), "index_build: buffer too small");
  TFRS_CHECK_ARG((reinterpret_cast<uintptr_t>(index_buf) & 15) == 0, "index_build: buffer must be 16-byte aligned");
  cudaStream_t st = (cudaStream_t)stream;
  IndexHeader h{};
  h.d = d; h.kb = (d + KSLAB - 1) / KSLAB; h.d_pad = h.kb * KSLAB; h.n = N; h.n_tiles = ceil_div(N, TILE_N);
  TFRS_CUDA(cudaMemsetAsync(index_buf, 0, HEADER_BYTES, st));
  header_kernel<<<1, 1, 0, st>>>(reinterpret_cast<IndexHeader*>(index_buf), h);
  TFRS_LAUNCH_CHECK();
  SideStats* cst = &reinterpret_cast<IndexHeader*>(index_buf)->st;
  const unsigned sgrid = (unsigned)(sm_count() * 8);
  corpus_stats_kernel<0><<<sgrid, 256, 0, st>>>(corpus, N, d, cst);
  TFRS_LAUNCH_CHECK();
  side_exp_kernel<<<1, 1, 0, st>>>(cst);
  TFRS_LAUNCH_CHECK();
  const long long s_tiles = norm_sample_tiles(N);
  if (s_tiles == 0) {
    corpus_stats_kernel<1><<<sgrid, 256, 0, st>>>(corpus, N, d, cst);
    TFRS_LAUNCH_CHECK();
  }
  auto image = [&](long long rows, long long tiles, unsigned char* dst, const int* rowmap) {
    const long long chunks = tiles * TILE_N * (long long)h.kb * 8;
    const unsigned blocks = (unsigned)(ceil_div(chunks, 256) < (1 << 20) ? ceil_div(chunks, 256) : (1 << 20));
    tile_image_kernel<<<blocks, 256, 0, st>>>(corpus, rows, d, h.kb, tiles, cst, dst, rowmap);
  };
  unsigned char* img = (unsigned char*)index_buf + HEADER_BYTES;
  image(N, h.n_tiles, img, nullptr);
  TFRS_LAUNCH_CHECK();
  if (s_tiles == 0) return TFRS_OK;

  // norm sample: the S rows of largest norm (ties to the lower index), their image, and phi -> header
  const long long S = s_tiles * TILE_N;
  const int nblk = (int)ceil_div(N, NS_CHUNK), nblk_s = (int)ceil_div(S, NS_CHUNK);
  const size_t o_rows = align_up((size_t)N * 4, 256), o_blk = o_rows + align_up((size_t)S * 4, 256);
  const size_t o_part = o_blk + align_up((size_t)nblk * 8, 256), o_sel = o_part + align_up((size_t)nblk * 8, 256);
  // probes: their rows, the exact top-(K+1) lists, the shares, the sample flags and the call's workspace
  Plan ppl;
  const bool probe_ok = make_plan(NORM_PROBES, N, d, NORM_PROBE_K + 1, ppl);
  const size_t pk = (size_t)NORM_PROBES * (NORM_PROBE_K + 1);
  const size_t o_probe = o_sel + align_up(sizeof(NormSelect), 256), o_ps = o_probe + align_up((size_t)NORM_PROBES * d * 4, 256);
  const size_t o_pi = o_ps + align_up(pk * 4, 256), o_share = o_pi + align_up(pk * 8, 256);
  const size_t o_flag = o_share + align_up((size_t)NORM_PROBES * 4, 256), o_pws = o_flag + align_up((size_t)N, 256);
  const size_t ws_bytes = probe_ok ? ppl.total + 16 : 0;
  unsigned char* scratch = nullptr;
  TFRS_CUDA(cudaMallocAsync((void**)&scratch, o_pws + ws_bytes, st));
  unsigned int* key = (unsigned int*)scratch;
  int* rowlist = (int*)(scratch + o_rows);
  int* blk = (int*)(scratch + o_blk);
  double* partial = (double*)(scratch + o_part);
  NormSelect* sel = (NormSelect*)(scratch + o_sel);
  int rc = TFRS_OK;
  // errors are recorded, not returned, so that the scratch memory is always freed
  auto launched = [&]() {
    count_launch();
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess && rc == TFRS_OK) { set_error("index_build: %s", cudaGetErrorString(e)); rc = TFRS_ERR_CUDA; }
  };
  if (cudaMemsetAsync(sel, 0, sizeof(NormSelect), st) != cudaSuccess) { set_error("index_build: memset failed"); rc = TFRS_ERR_CUDA; }
  corpus_stats_kernel<1><<<sgrid, 256, 0, st>>>(corpus, N, d, cst, key);
  launched();
  for (int bit = 31; bit >= 0; --bit) { norm_select_count_kernel<<<sgrid, 256, 0, st>>>(key, N, S, bit, sel); launched(); }
  norm_select_chunks_kernel<<<nblk, 256, 0, st>>>(key, N, S, sel, blk);
  launched();
  norm_select_offsets_kernel<<<1, 1, 0, st>>>(blk, nblk, S, sel);
  launched();
  norm_select_write_kernel<<<nblk, 256, 0, st>>>(key, N, S, sel, blk, rowlist);
  launched();
  image(S, s_tiles, img + h.n_tiles * h.kb * (long long)SLAB_BYTES, rowlist);
  launched();
  norm_phi_init_kernel<<<1, 1, 0, st>>>(sel, cst);
  launched();
  IndexHeader* hdr = reinterpret_cast<IndexHeader*>(index_buf);
  for (int it = 0; it < 48; ++it) {   // bracket [0, 40 max|c|] / 2^48
    norm_phi_partial_kernel<<<nblk, 256, 0, st>>>(key, nullptr, N, sel, partial);
    launched();
    norm_phi_step_kernel<<<1, 1, 0, st>>>(partial, nblk, N, 0, sel, hdr, nullptr);
    launched();
  }
  float* share = (float*)(scratch + o_share);
  if (cudaMemsetAsync(share, 0, (size_t)NORM_PROBES * 4, st) != cudaSuccess && rc == TFRS_OK) { set_error("index_build: memset failed"); rc = TFRS_ERR_CUDA; }
  if (probe_ok && rc == TFRS_OK) {
    unsigned char* flags = scratch + o_flag;
    if (cudaMemsetAsync(flags, 0, (size_t)N, st) != cudaSuccess) { set_error("index_build: memset failed"); rc = TFRS_ERR_CUDA; }
    norm_sample_flags_kernel<<<sgrid, 256, 0, st>>>(rowlist, S, flags);
    launched();
    float* probes = (float*)(scratch + o_probe);
    norm_probe_gather_kernel<<<NORM_PROBES, 32, 0, st>>>(corpus, N, d, probes);
    launched();
    // the header still says SAMPLE_STRIDED: an exact call on the strided-sample path
    Call c{};
    c.mode = FIN_TOPK; c.q = probes; c.Q = NORM_PROBES; c.corpus = corpus; c.index_buf = index_buf; c.N = N; c.d = d;
    c.k = NORM_PROBE_K + 1; c.ws = scratch + o_pws; c.ws_bytes = ws_bytes; c.st = st;
    c.out_s = (float*)(scratch + o_ps); c.out_i = (long long*)(scratch + o_pi);
    const int prc = run_call(c);
    if (prc != TFRS_OK && rc == TFRS_OK) rc = prc;
    norm_probe_share_kernel<<<NORM_PROBES, 32, 0, st>>>(c.out_i, N, flags, share);
    launched();
  }
  norm_phi_partial_kernel<<<nblk_s, 256, 0, st>>>(key, rowlist, S, sel, partial);
  launched();
  norm_phi_step_kernel<<<1, 1, 0, st>>>(partial, nblk_s, N, 1, sel, hdr, share);
  launched();
  const cudaError_t fe = cudaFreeAsync(scratch, st);
  if (fe != cudaSuccess && rc == TFRS_OK) { set_error("index_build: %s", cudaGetErrorString(fe)); rc = TFRS_ERR_CUDA; }
  return rc;
}

extern "C" size_t tfrs_topk_tc_workspace_bytes(int64_t Q, int64_t N, int d, int k) {
  Plan pl;
  if (!make_plan(Q, N, d, k, pl)) return 0;
  return pl.total + 16;
}

extern "C" int tfrs_topk_tc_f32(const float* q, int64_t Q, const float* corpus, const void* index_buf, int64_t N, int d,
                                int k, int64_t index_offset, float* out_scores, int64_t* out_idx, void* ws, size_t ws_bytes,
                                void* stream) {
  TFRS_CHECK_ARG(q && corpus && index_buf && out_scores && out_idx, "topk_tc: NULL pointer");
  TFRS_CHECK_ARG(k <= N, "input must have at least k columns. Had %lld, needed %d", (long long)N, k);
  Call c{};
  c.mode = FIN_TOPK; c.q = q; c.Q = Q; c.corpus = corpus; c.index_buf = index_buf; c.N = N; c.d = d; c.k = k;
  c.index_offset = index_offset; c.ws = ws; c.ws_bytes = ws_bytes; c.st = (cudaStream_t)stream;
  c.out_s = out_scores; c.out_i = (long long*)out_idx;
  return run_call(c);
}

// internal (comm.cu): the local scan of the sharded call, with the threshold hook and short lists allowed
int tfrs::tc_topk_sharded_local(const float* q, int64_t Q, const float* corpus, const void* index_buf, int64_t N, int d, int k,
                                int64_t index_offset, float* out_scores, int64_t* out_idx, void* ws, size_t ws_bytes, void* stream,
                                tfrs::ThrHook hook, void* hook_ctx) {
  Call c{};
  c.mode = FIN_TOPK; c.q = q; c.Q = Q; c.corpus = corpus; c.index_buf = index_buf; c.N = N; c.d = d; c.k = k;
  c.index_offset = index_offset; c.ws = ws; c.ws_bytes = ws_bytes; c.st = (cudaStream_t)stream;
  c.out_s = out_scores; c.out_i = (long long*)out_idx;
  c.hook = hook; c.hook_ctx = hook_ctx; c.allow_short = hook ? 1 : 0;
  return run_call(c);
}

extern "C" int tfrs_topk_tc_exclude_f32(const float* q, int64_t Q, const float* corpus, const void* index_buf, int64_t N, int d,
                                        int k, int64_t index_offset, const int64_t* identifiers, const int64_t* exclusions,
                                        int n_excl, float* out_scores, int64_t* out_idx, void* ws, size_t ws_bytes, void* stream) {
  TFRS_CHECK_ARG(q && corpus && index_buf && out_scores && out_idx && exclusions && n_excl > 0, "topk_tc_exclude: bad argument");
  TFRS_CHECK_ARG((long long)k + n_excl <= N, "input must have at least k columns. Had %lld, needed %d", (long long)N, k + n_excl);
  Call c{};
  c.mode = FIN_EXCLUDE; c.q = q; c.Q = Q; c.corpus = corpus; c.index_buf = index_buf; c.N = N; c.d = d; c.k = k + n_excl;
  c.index_offset = index_offset; c.ws = ws; c.ws_bytes = ws_bytes; c.st = (cudaStream_t)stream;
  c.out_s = out_scores; c.out_i = (long long*)out_idx;
  c.identifiers = (const long long*)identifiers; c.exclusions = (const long long*)exclusions; c.n_excl = n_excl; c.k_out = k;
  return run_call(c);
}

extern "C" int tfrs_topk_tc_count_f32(const float* q, int64_t Q, const float* corpus, const void* index_buf, int64_t N, int d,
                                      int k, const float* positive_scores, int32_t* out_count, void* ws, size_t ws_bytes,
                                      void* stream) {
  TFRS_CHECK_ARG(q && corpus && index_buf && positive_scores && out_count, "topk_tc_count: NULL pointer");
  TFRS_CHECK_ARG(k <= N, "input must have at least k columns. Had %lld, needed %d", (long long)N, k);
  Call c{};
  c.mode = FIN_COUNT; c.q = q; c.Q = Q; c.corpus = corpus; c.index_buf = index_buf; c.N = N; c.d = d; c.k = k;
  c.ws = ws; c.ws_bytes = ws_bytes; c.st = (cudaStream_t)stream;
  c.pos = positive_scores; c.out_count = out_count;
  return run_call(c);
}

// Debug/test introspection: where the per-query survivor counts / fallback flags of the last call live
// inside the caller's workspace (byte offsets from the 16-byte-aligned workspace base).
extern "C" int tfrs_topk_tc_layout(int64_t Q, int64_t N, int d, int k, int64_t* out10) {
  TFRS_CHECK_ARG(out10, "topk_tc_layout: NULL pointer");
  Plan pl;
  if (!make_plan(Q, N, d, k, pl)) { set_error("topk_tc_layout: unsupported shape"); return TFRS_ERR_UNSUPPORTED; }
  out10[0] = (int64_t)pl.o_count; out10[1] = (int64_t)pl.o_ovf; out10[2] = (int64_t)pl.o_thr; out10[3] = (int64_t)pl.o_cand;
  out10[4] = pl.parts_full * 2; out10[5] = pl.cap_part; out10[6] = pl.Qp; out10[7] = (int64_t)pl.o_cut;
  out10[8] = pl.n_bins; out10[9] = (int64_t)pl.o_qexp;
  return TFRS_OK;
}

// The same for the two-threshold filter: where thr_safe and the per-row retry marks live, the bin rank of the filter
// threshold of a TOPK / EXCLUDE call and the sample stride it was derived from.
extern "C" int tfrs_topk_tc_retry_layout(int64_t Q, int64_t N, int d, int k, int64_t* out4) {
  TFRS_CHECK_ARG(out4, "topk_tc_retry_layout: NULL pointer");
  Plan pl;
  if (!make_plan(Q, N, d, k, pl)) { set_error("topk_tc_retry_layout: unsupported shape"); return TFRS_ERR_UNSUPPORTED; }
  out4[0] = (int64_t)pl.o_thr_safe; out4[1] = (int64_t)pl.o_retry; out4[2] = pl.k_filter; out4[3] = pl.stride;
  return TFRS_OK;
}

// The sampled pass on a norm-sample index: where the bin maxima and margins live, and how the bins are laid out.
extern "C" int tfrs_topk_tc_sample_layout(int64_t Q, int64_t N, int d, int k, int64_t* out8) {
  TFRS_CHECK_ARG(out8, "topk_tc_sample_layout: NULL pointer");
  Plan pl;
  if (!make_plan(Q, N, d, k, pl)) { set_error("topk_tc_sample_layout: unsupported shape"); return TFRS_ERR_UNSUPPORTED; }
  out8[0] = (int64_t)pl.o_binmax; out8[1] = pl.bins_ld; out8[2] = pl.n_bins_norm; out8[3] = pl.group_norm;
  out8[4] = pl.bins_per_part_norm; out8[5] = pl.parts_sample; out8[6] = pl.n_seq_norm; out8[7] = (int64_t)pl.o_margin;
  return TFRS_OK;
}

extern "C" int tfrs_profile_enable(int on) {
  g_prof.on = on != 0;
  g_prof.calls = 0;
  return TFRS_OK;
}

// Synchronises the device, then returns the summed stage times (ms) over the calls recorded since
// tfrs_profile_enable(1): stage_ms[0..3] = prep, sample+threshold, filter, finalize+fallback.
extern "C" int tfrs_profile_read(float* stage_ms, int* calls) {
  TFRS_CHECK_ARG(stage_ms && calls, "profile_read: NULL pointer");
  TFRS_CUDA(cudaDeviceSynchronize());
  for (int s = 0; s < 4; ++s) stage_ms[s] = 0.f;
  for (int c = 0; c < g_prof.calls; ++c)
    for (int s = 0; s < 4; ++s) {
      float ms = 0.f;
      TFRS_CUDA(cudaEventElapsedTime(&ms, g_prof.ev[c][s], g_prof.ev[c][s + 1]));
      stage_ms[s] += ms;
    }
  *calls = g_prof.calls;
  return TFRS_OK;
}
