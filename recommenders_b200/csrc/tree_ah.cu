// tree_ah.cu -- K9: tree-AH approximate retrieval (partitioned asymmetric hashing), the algorithm of ScaNN's
// factorized_top_k.ScaNN (layers/factorized_top_k.py:613-796) with the rules pinned in DESIGN.md §2.
//
// Index build (not the hot path; the host drives the Lloyd iterations):
//   tfrs_tree_ah_assign_f32           nearest center by squared L2 = top-1 of [x, 1] . [c, -0.5|c|^2] (tfrs_topk_scan_f32)
//   tfrs_tree_ah_group                leaf-major order: K4's (id, position) bitonic sort, then leaf offsets
//   tfrs_tree_ah_update_centroids_f32 ordered float64 mean of every leaf's members
//   tfrs_tree_ah_init_codebooks_f32   / _update_codebooks_f32 / tfrs_tree_ah_encode: the 16-center codebooks of the
//                                     residuals x - c_leaf(x), block by block, and the packed 4-bit codes
// Search (hot path), per chunk of queries:
//   probe scan (tfrs_topk_scan_f32 over the centroids) -> int8 LUTs (ta_lut) -> AH scan + pre-selection
//   (row_topk_kernel<AhProvider>, one CTA per (query, probed leaf, slice)) -> sorted-list merge -> optional exact
//   rescore of the k' survivors (row_topk_kernel<RescoreProvider>) -> padding to (NaN, 0) (ta_finalize).
#include "adagrad.cuh"
#include "rowselect.cuh"

namespace tfrs {

constexpr long long TA_ASSIGN_ROWS = 65536;   // rows per assignment scan call
constexpr int TA_MAX_D = 256, TA_MAX_DPB = 8, TA_MAX_K = 2048;
constexpr long long TA_MAX_N = 1ll << 24;     // row positions travel in the low 24 bits of K4's sort keys
constexpr size_t TA_SEARCH_BUDGET = (size_t)512 << 20;

static inline int ta_blocks(int d, int dpb) { return (d + dpb - 1) / dpb; }
static inline int ta_words(int B) { return (B + 7) / 8; }

// warp per row: out row = [x, 1] (mode 0) or [x, -0.5f * canonical |x|^2] (mode 1)
__global__ void __launch_bounds__(256)
ta_augment(const float* __restrict__ x, long long n, int d, int mode, float* __restrict__ out) {
  const long long r = ((long long)blockIdx.x * 256 + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (r >= n) return;
  const float* xr = x + r * d;
  float* o = out + r * (d + 1);
  for (int c = lane; c < d; c += 32) o[c] = xr[c];
  if (lane == 0) {
    float last = 1.f;
    if (mode) {
      float acc = 0.f;
      for (int c = 0; c < d; ++c) acc = fmaf(xr[c], xr[c], acc);
      last = __fmul_rn(-0.5f, acc);
    }
    o[d] = last;
  }
}

__global__ void __launch_bounds__(256)
ta_order(const unsigned long long* __restrict__ keys, long long n, int* __restrict__ order) {
  const long long i = (long long)blockIdx.x * 256 + threadIdx.x;
  if (i < n) order[i] = (int)(keys[i] & 0xFFFFFFull);
}

// offsets[l] = first sorted slot whose leaf is >= l
__global__ void __launch_bounds__(256)
ta_offsets(const unsigned long long* __restrict__ keys, long long n, int L, int* __restrict__ offsets) {
  const int l = blockIdx.x * 256 + threadIdx.x;
  if (l > L) return;
  long long lo = 0, hi = n;
  while (lo < hi) { const long long mid = (lo + hi) >> 1; if ((long long)(keys[mid] >> 24) < l) lo = mid + 1; else hi = mid; }
  offsets[l] = (int)lo;
}

// thread per (leaf, column): the members in ascending position order, summed sequentially in float64 (the first member
// starts the sum, so a sum of -0.0s stays -0.0), divided once and rounded to fp32; an empty leaf keeps its centroid
__global__ void __launch_bounds__(256)
ta_update_centroids(const float* __restrict__ x, int d, const int* __restrict__ order, const int* __restrict__ offsets,
                    int L, float* __restrict__ cent) {
  const long long t = (long long)blockIdx.x * 256 + threadIdx.x;
  if (t >= (long long)L * d) return;
  const int l = (int)(t / d), c = (int)(t - (long long)l * d);
  const int b = offsets[l], e = offsets[l + 1];
  if (b == e) return;
  double s = (double)x[(long long)order[b] * d + c];
#pragma unroll 8
  for (int m = b + 1; m < e; ++m) s += (double)x[(long long)order[m] * d + c];
  cent[t] = (float)(s / (double)(e - b));
}

// codebooks [B][16][dpb] (the last block's unused dims are 0): center j of every block = the residual of training
// position pos[j]
__global__ void __launch_bounds__(256)
ta_init_codebooks(const float* __restrict__ x, int d, const long long* __restrict__ pos, const long long* __restrict__ leaf,
                  const float* __restrict__ cent, int dpb, int B, float* __restrict__ cb) {
  const int t = blockIdx.x * 256 + threadIdx.x;
  if (t >= B * 16 * dpb) return;
  const int b = t / (16 * dpb), j = (t / dpb) & 15, u = t % dpb, c = b * dpb + u;
  float v = 0.f;
  if (c < d) {
    const long long p = pos[j];
    v = __fsub_rn(x[p * d + c], cent[leaf[p] * d + c]);
  }
  cb[t] = v;
}

// codes of position p (row = rows ? rows[p] : p): per block the top-1 of [r_b, 1] . [cb_j, -0.5f |cb_j|^2] over the 16
// centers, ties to the lower j; 8 codes per uint32 word (block 8w + e in bits 4e..4e+3), W words per position
__global__ void __launch_bounds__(256)
ta_encode(const float* __restrict__ x, int d, const int* __restrict__ rows, long long n, const long long* __restrict__ leaf,
          const float* __restrict__ cent, const float* __restrict__ cb, int dpb, int B, int W, uint32_t* __restrict__ codes) {
  extern __shared__ float ta_cb[];   // [B*16*dpb] centers, then [B*16] biases
  float* bias = ta_cb + B * 16 * dpb;
  for (int t = threadIdx.x; t < B * 16 * dpb; t += 256) ta_cb[t] = cb[t];
  __syncthreads();
  for (int e = threadIdx.x; e < B * 16; e += 256) {
    const int b = e >> 4, w = min(dpb, d - b * dpb);
    float acc = 0.f;
    for (int u = 0; u < w; ++u) acc = fmaf(ta_cb[e * dpb + u], ta_cb[e * dpb + u], acc);
    bias[e] = __fmul_rn(-0.5f, acc);
  }
  __syncthreads();
  const long long t = (long long)blockIdx.x * 256 + threadIdx.x;
  if (t >= n * W) return;
  const long long p = t / W;
  const int wd = (int)(t - p * W);
  const long long row = rows ? (long long)rows[p] : p;
  const float* xr = x + row * d;
  const float* cr = cent + leaf[row] * d;
  uint32_t word = 0;
  for (int e = 0; e < 8; ++e) {
    const int b = wd * 8 + e;
    if (b >= B) break;
    const int w = min(dpb, d - b * dpb);
    float r[TA_MAX_DPB];
#pragma unroll
    for (int u = 0; u < TA_MAX_DPB; ++u) r[u] = u < w ? __fsub_rn(xr[b * dpb + u], cr[b * dpb + u]) : 0.f;
    float best = 0.f;
    int bj = 0;
    for (int j = 0; j < 16; ++j) {
      const float* cj = ta_cb + (b * 16 + j) * dpb;
      float acc = 0.f;
#pragma unroll
      for (int u = 0; u < TA_MAX_DPB; ++u) if (u < w) acc = fmaf(r[u], cj[u], acc);
      acc = __fadd_rn(acc, bias[b * 16 + j]);
      if (j == 0 || acc > best) { best = acc; bj = j; }
    }
    word |= (uint32_t)bj << (4 * e);
  }
  codes[t] = word;
}

// thread per (block, center, dim): the residuals of the training positions coded j in block b, in ascending position
// order, float64 as ta_update_centroids; a center without members keeps its value
__global__ void __launch_bounds__(256)
ta_update_codebooks(const float* __restrict__ x, int d, long long n, const long long* __restrict__ leaf,
                    const float* __restrict__ cent, const uint32_t* __restrict__ codes, int W, int dpb, int B,
                    float* __restrict__ cb) {
  const int t = blockIdx.x * 256 + threadIdx.x;
  if (t >= B * 16 * dpb) return;
  const int b = t / (16 * dpb), j = (t / dpb) & 15, u = t % dpb, c = b * dpb + u;
  if (c >= d) return;
  const int wd = b >> 3, sh = (b & 7) * 4;
  double s = 0.0;
  long long cnt = 0;
#pragma unroll 4
  for (long long i = 0; i < n; ++i) {
    if ((int)((__ldg(codes + i * W + wd) >> sh) & 15u) != j) continue;
    const double v = (double)__fsub_rn(__ldg(x + i * d + c), __ldg(cent + leaf[i] * d + c));
    s = cnt ? s + v : v;
    ++cnt;
  }
  if (cnt) cb[t] = (float)(s / (double)cnt);
}

// one CTA per query: T[b][j] = canonical dot of the query's block b with center j; s = max|T| / 127 (0 when max|T| = 0);
// LUT = (int8) rint(T / s), W*8 blocks of 16 bytes per query (blocks >= B are 0)
__global__ void __launch_bounds__(256)
ta_lut(const float* __restrict__ q, int d, const float* __restrict__ cb, int dpb, int B, int W, int8_t* __restrict__ lut,
       float* __restrict__ scale) {
  __shared__ float T[TA_MAX_D * 16];
  __shared__ float red[8];
  const long long qi = blockIdx.x;
  const float* qr = q + qi * d;
  float m = 0.f;
  for (int e = threadIdx.x; e < B * 16; e += 256) {
    const int b = e >> 4, w = min(dpb, d - b * dpb);
    float acc = 0.f;
    for (int u = 0; u < w; ++u) acc = fmaf(qr[b * dpb + u], cb[e * dpb + u], acc);
    T[e] = acc;
    m = fmaxf(m, fabsf(acc));
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = m;
  __syncthreads();
  m = red[0];
  for (int w = 1; w < 8; ++w) m = fmaxf(m, red[w]);
  const float s = m > 0.f ? __fdiv_rn(m, 127.f) : 0.f;
  int8_t* out = lut + qi * W * 128;
  for (int e = threadIdx.x; e < W * 128; e += 256)
    out[e] = (e < B * 16 && s != 0.f) ? (int8_t)__float2int_rn(__fdiv_rn(T[e], s)) : (int8_t)0;
  if (threadIdx.x == 0) scale[qi] = s;
}

// One rowselect row = (query q, probed leaf p, slice s of that leaf), numbered row = (p*S + s) * Qc + q so that the
// output lists are laid out [list][query][k'] for the sorted-list merge.  A slice shorter than k' is padded with
// (-inf, INT64_MAX), so every list has exactly k' sorted entries.
struct AhProvider {
  const int8_t* lut; const float* scale; const float* probe_s; const long long* probe_leaf;
  const int* offsets; const uint32_t* codes; const int* order;
  int Qc, P, S, W, kp;
  const int8_t* sl; long long lo; int n; float dot, sc;   // this row's, set by begin()
  __device__ void begin(int row, void* extra) {
    const int q = row % Qc, l = row / Qc, p = l / S, s = l - p * S;
    const long long leaf = probe_leaf[(long long)q * P + p];
    const int b = offsets[leaf], size = offsets[leaf + 1] - b;
    lo = b + (long long)size * s / S;
    n = (int)(b + (long long)size * (s + 1) / S - lo);
    dot = probe_s[(long long)q * P + p];
    sc = scale[q];
    int* sm = reinterpret_cast<int*>(extra);
    const int* src = reinterpret_cast<const int*>(lut + (long long)q * W * 128);
    for (int t = threadIdx.x; t < W * 32; t += blockDim.x) sm[t] = src[t];
    sl = reinterpret_cast<const int8_t*>(extra);
  }
  __device__ long long count(int) const { return n > kp ? n : kp; }
  __device__ void get(int, long long t, float& s, long long& i) const {
    if (t >= n) { s = -INFINITY; i = LLONG_MAX; return; }
    const long long pos = lo + t;
    const uint32_t* cw = codes + pos * W;
    int acc = 0;
    for (int w = 0; w < W; ++w) {
      const uint32_t v = __ldg(cw + w);
      const int8_t* lw = sl + w * 128;   // lanes read the same block's 16 bytes: at most 4 banks, no conflict
#pragma unroll
      for (int e = 0; e < 8; ++e) acc += lw[e * 16 + ((v >> (4 * e)) & 15u)];
    }
    s = __fadd_rn(dot, __fmul_rn(sc, (float)acc));
    i = order[pos];
  }
};

// exact rescore of the k' pre-selected rows of every query (row = query of the chunk); padding stays padding
struct RescoreProvider {
  const float* q; const float* rows; const float* cs; const long long* ci; int d, kp;
  __device__ void begin(int, void*) {}
  __device__ long long count(int) const { return kp; }
  __device__ void get(int row, long long t, float& s, long long& i) const {
    i = ci[(long long)row * kp + t];
    if (i == LLONG_MAX) { s = -INFINITY; return; }
    const float* qr = q + (long long)row * d;
    const float* xr = rows + i * d;
    float acc = 0.f;
    for (int c = 0; c < d; ++c) acc = fmaf(qr[c], __ldg(xr + c), acc);
    s = acc;
  }
};

__global__ void __launch_bounds__(256)
ta_finalize(const float* __restrict__ s, const long long* __restrict__ i, long long n, float* __restrict__ out_s,
            int64_t* __restrict__ out_i) {
  const long long t = (long long)blockIdx.x * 256 + threadIdx.x;
  if (t >= n) return;
  const long long v = i[t];
  out_s[t] = v == LLONG_MAX ? __int_as_float(0x7fc00000) : s[t];
  out_i[t] = v == LLONG_MAX ? 0 : v;
}

struct TaPlan {
  int S; long long qc;
  size_t lists_s, lists_i, merged_s, merged_i, lut, scale, probe_s, probe_i, resc_s, resc_i, scan, total;
};

// Slices per (query, leaf): enough CTAs for two waves when Q * P is small (Q = 1), never slices under 256 rows.
// Queries are chunked so that the Q x P x S lists of k' entries stay within TA_SEARCH_BUDGET.
static TaPlan ta_plan(long long Q, int d, int L, int P, int B, int k, int kp, int reorder, long long N) {
  TaPlan p;
  const long long want = ceil_div(2ll * sm_count(), Q * P);
  const long long by_rows = (N / L) / 256;
  long long S = want < by_rows ? want : by_rows;
  if (S > 64) S = 64;
  if (S < 1) S = 1;
  p.S = (int)S;
  const int W = ta_words(B);
  const size_t per_q = (size_t)P * S * kp * 12 + (size_t)kp * 12 + (size_t)W * 128 + 4 + (size_t)P * 12 +
                       (reorder ? (size_t)k * 12 : 0) + (size_t)P * 24;
  long long qc = (long long)(TA_SEARCH_BUDGET / per_q);
  if (qc < 1) qc = 1;
  if (qc > Q) qc = Q;
  p.qc = qc;
  p.lists_s = align_up((size_t)qc * P * S * kp * 4, 256);
  p.lists_i = align_up((size_t)qc * P * S * kp * 8, 256);
  p.merged_s = align_up((size_t)qc * kp * 4, 256);
  p.merged_i = align_up((size_t)qc * kp * 8, 256);
  p.lut = align_up((size_t)qc * W * 128, 256);
  p.scale = align_up((size_t)qc * 4, 256);
  p.probe_s = align_up((size_t)qc * P * 4, 256);
  p.probe_i = align_up((size_t)qc * P * 8, 256);
  p.resc_s = reorder ? align_up((size_t)qc * k * 4, 256) : 0;
  p.resc_i = reorder ? align_up((size_t)qc * k * 8, 256) : 0;
  p.scan = tfrs_topk_scan_workspace_bytes(qc, L, d, P);
  p.total = p.lists_s + p.lists_i + p.merged_s + p.merged_i + p.lut + p.scale + p.probe_s + p.probe_i + p.resc_s +
            p.resc_i + p.scan;
  return p;
}

}  // namespace tfrs

using namespace tfrs;

extern "C" size_t tfrs_tree_ah_assign_workspace_bytes(int64_t n, int d, int L) {
  const long long qc = n < TA_ASSIGN_ROWS ? (n > 0 ? n : 1) : TA_ASSIGN_ROWS;
  return align_up((size_t)L * (d + 1) * 4, 256) + align_up((size_t)qc * (d + 1) * 4, 256) + align_up((size_t)qc * 4, 256) +
         tfrs_topk_scan_workspace_bytes(qc, L, d + 1, 1);
}

extern "C" int tfrs_tree_ah_assign_f32(const float* x, int64_t n, int d, const float* centers, int L, int64_t* leaf,
                                       void* ws, size_t ws_bytes, void* stream) {
  TFRS_CHECK_ARG(n >= 0 && d >= 1 && d <= TA_MAX_D && L >= 1, "tree_ah_assign: bad shape n=%lld d=%d L=%d", (long long)n, d, L);
  if (n == 0) return TFRS_OK;
  TFRS_CHECK_ARG(x && centers && leaf, "tree_ah_assign: NULL pointer");
  const size_t need = tfrs_tree_ah_assign_workspace_bytes(n, d, L);
  if (!ws || ws_bytes < need) { set_error("tree_ah_assign: workspace too small (%zu < %zu)", ws_bytes, need); return TFRS_ERR_WORKSPACE_TOO_SMALL; }
  cudaStream_t st = (cudaStream_t)stream;
  const long long qc = n < TA_ASSIGN_ROWS ? n : TA_ASSIGN_ROWS;
  unsigned char* w = (unsigned char*)ws;
  float* ac = (float*)w; w += align_up((size_t)L * (d + 1) * 4, 256);
  float* ax = (float*)w; w += align_up((size_t)qc * (d + 1) * 4, 256);
  float* sc = (float*)w; w += align_up((size_t)qc * 4, 256);
  const size_t scan_bytes = tfrs_topk_scan_workspace_bytes(qc, L, d + 1, 1);
  ta_augment<<<(unsigned)ceil_div((long long)L * 32, 256), 256, 0, st>>>(centers, L, d, 1, ac);
  TFRS_LAUNCH_CHECK();
  for (long long r0 = 0; r0 < n; r0 += qc) {
    const long long m = (n - r0) < qc ? (n - r0) : qc;
    ta_augment<<<(unsigned)ceil_div(m * 32, 256), 256, 0, st>>>(x + r0 * d, m, d, 0, ax);
    TFRS_LAUNCH_CHECK();
    const int rc = tfrs_topk_scan_f32(ax, m, ac, L, d + 1, 1, 0, nullptr, nullptr, 0, sc, leaf + r0, w, scan_bytes, stream);
    if (rc) return rc;
  }
  return TFRS_OK;
}

extern "C" size_t tfrs_tree_ah_group_workspace_bytes(int64_t n) { return ag_group_workspace_bytes(n); }

extern "C" int tfrs_tree_ah_group(const int64_t* leaf, int64_t n, int L, int32_t* offsets, int32_t* order, void* ws,
                                  size_t ws_bytes, void* stream) {
  TFRS_CHECK_ARG(n >= 1 && n < TA_MAX_N && L >= 1, "tree_ah_group: n=%lld must be in [1, 2^24), L=%d >= 1", (long long)n, L);
  TFRS_CHECK_ARG(leaf && offsets && order, "tree_ah_group: NULL pointer");
  if (!ws || ws_bytes < ag_group_workspace_bytes(n)) { set_error("tree_ah_group: workspace too small"); return TFRS_ERR_WORKSPACE_TOO_SMALL; }
  cudaStream_t st = (cudaStream_t)stream;
  const int rc = ag_sort(leaf, TFRS_I64, n, L, ws, st);
  if (rc) return rc;
  const unsigned long long* keys = (const unsigned long long*)ws;
  ta_order<<<(unsigned)ceil_div(n, 256), 256, 0, st>>>(keys, n, order);
  TFRS_LAUNCH_CHECK();
  ta_offsets<<<(unsigned)ceil_div(L + 1, 256), 256, 0, st>>>(keys, n, L, offsets);
  TFRS_LAUNCH_CHECK();
  return TFRS_OK;
}

extern "C" int tfrs_tree_ah_update_centroids_f32(const float* x, int d, const int32_t* order, const int32_t* offsets, int L,
                                                 float* centroids, void* stream) {
  TFRS_CHECK_ARG(d >= 1 && d <= TA_MAX_D && L >= 1, "tree_ah_update_centroids: bad shape");
  TFRS_CHECK_ARG(x && order && offsets && centroids, "tree_ah_update_centroids: NULL pointer");
  ta_update_centroids<<<(unsigned)ceil_div((long long)L * d, 256), 256, 0, (cudaStream_t)stream>>>(x, d, order, offsets, L,
                                                                                                    centroids);
  TFRS_LAUNCH_CHECK();
  return TFRS_OK;
}

extern "C" int tfrs_tree_ah_init_codebooks_f32(const float* x, int d, const int64_t* pos, const int64_t* leaf,
                                               const float* centroids, int dpb, float* codebooks, void* stream) {
  TFRS_CHECK_ARG(d >= 1 && d <= TA_MAX_D && dpb >= 1 && dpb <= TA_MAX_DPB, "tree_ah_init_codebooks: bad shape");
  TFRS_CHECK_ARG(x && pos && leaf && centroids && codebooks, "tree_ah_init_codebooks: NULL pointer");
  const int B = ta_blocks(d, dpb);
  ta_init_codebooks<<<(unsigned)ceil_div(B * 16 * dpb, 256), 256, 0, (cudaStream_t)stream>>>(
      x, d, (const long long*)pos, (const long long*)leaf, centroids, dpb, B, codebooks);
  TFRS_LAUNCH_CHECK();
  return TFRS_OK;
}

extern "C" int tfrs_tree_ah_encode(const float* x, int d, const int32_t* rows, int64_t n, const int64_t* leaf,
                                   const float* centroids, const float* codebooks, int dpb, uint32_t* codes, void* stream) {
  TFRS_CHECK_ARG(n >= 0 && d >= 1 && d <= TA_MAX_D && dpb >= 1 && dpb <= TA_MAX_DPB, "tree_ah_encode: bad shape");
  if (n == 0) return TFRS_OK;
  TFRS_CHECK_ARG(x && leaf && centroids && codebooks && codes, "tree_ah_encode: NULL pointer");
  const int B = ta_blocks(d, dpb), W = ta_words(B);
  const size_t smem = (size_t)B * 16 * (dpb + 1) * 4;
  TFRS_DYN_SMEM(ta_encode, 48 * 1024);
  ta_encode<<<(unsigned)ceil_div(n * W, 256), 256, smem, (cudaStream_t)stream>>>(
      x, d, rows, n, (const long long*)leaf, centroids, codebooks, dpb, B, W, codes);
  TFRS_LAUNCH_CHECK();
  return TFRS_OK;
}

extern "C" int tfrs_tree_ah_update_codebooks_f32(const float* x, int d, int64_t n, const int64_t* leaf,
                                                 const float* centroids, const uint32_t* codes, int dpb, float* codebooks,
                                                 void* stream) {
  TFRS_CHECK_ARG(n >= 1 && d >= 1 && d <= TA_MAX_D && dpb >= 1 && dpb <= TA_MAX_DPB, "tree_ah_update_codebooks: bad shape");
  TFRS_CHECK_ARG(x && leaf && centroids && codes && codebooks, "tree_ah_update_codebooks: NULL pointer");
  const int B = ta_blocks(d, dpb);
  ta_update_codebooks<<<(unsigned)ceil_div(B * 16 * dpb, 256), 256, 0, (cudaStream_t)stream>>>(
      x, d, n, (const long long*)leaf, centroids, codes, ta_words(B), dpb, B, codebooks);
  TFRS_LAUNCH_CHECK();
  return TFRS_OK;
}

extern "C" size_t tfrs_tree_ah_search_workspace_bytes(int64_t Q, int d, int L, int P, int dpb, int k, int kp, int reorder,
                                                      int64_t N) {
  if (Q <= 0 || d < 1 || dpb < 1 || L < 1 || P < 1 || kp < 1 || N < 1) return 256;
  return ta_plan(Q, d, L, P, ta_blocks(d, dpb), k, kp, reorder, N).total;
}

extern "C" int tfrs_tree_ah_search_f32(const float* q, int64_t Q, int d, const float* centroids, int L,
                                       const int32_t* leaf_offsets, const float* codebooks, int dpb, const uint32_t* codes,
                                       const int32_t* order, int64_t N, const float* rows, int P, int k, int kp,
                                       float* out_scores, int64_t* out_idx, void* ws, size_t ws_bytes, void* stream) {
  TFRS_CHECK_ARG(Q >= 0 && Q < (1ll << 31) && d >= 1 && d <= TA_MAX_D && dpb >= 1 && dpb <= TA_MAX_DPB,
                 "tree_ah_search: bad shape Q=%lld d=%d dpb=%d", (long long)Q, d, dpb);
  TFRS_CHECK_ARG(N >= 1 && N < TA_MAX_N && L >= 1 && L <= N, "tree_ah_search: bad index N=%lld L=%d", (long long)N, L);
  TFRS_CHECK_ARG(P >= 1 && P <= L && P <= TA_MAX_K, "tree_ah_search: P=%d must be in [1, min(L, 2048)]", P);
  TFRS_CHECK_ARG(k >= 1 && k <= kp && kp <= TA_MAX_K, "tree_ah_search: need 1 <= k=%d <= k'=%d <= 2048", k, kp);
  TFRS_CHECK_ARG(rows || kp == k, "tree_ah_search: k' > k needs the reordering rows");
  if (Q == 0) return TFRS_OK;
  TFRS_CHECK_ARG(q && centroids && leaf_offsets && codebooks && codes && order && out_scores && out_idx,
                 "tree_ah_search: NULL pointer");
  const int reorder = rows != nullptr;
  const int B = ta_blocks(d, dpb), W = ta_words(B);
  const TaPlan p = ta_plan(Q, d, L, P, B, k, kp, reorder, N);
  if (!ws || ws_bytes < p.total) { set_error("tree_ah_search: workspace too small (%zu < %zu)", ws_bytes, p.total); return TFRS_ERR_WORKSPACE_TOO_SMALL; }
  cudaStream_t st = (cudaStream_t)stream;
  unsigned char* w = (unsigned char*)ws;
  float* lists_s = (float*)w; w += p.lists_s;
  long long* lists_i = (long long*)w; w += p.lists_i;
  float* merged_s = (float*)w; w += p.merged_s;
  long long* merged_i = (long long*)w; w += p.merged_i;
  int8_t* lut = (int8_t*)w; w += p.lut;
  float* scale = (float*)w; w += p.scale;
  float* probe_s = (float*)w; w += p.probe_s;
  long long* probe_i = (long long*)w; w += p.probe_i;
  float* resc_s = (float*)w; w += p.resc_s;
  long long* resc_i = (long long*)w; w += p.resc_i;
  void* scan_ws = w;

  const int cap_a = rowselect_cap(kp), cap_r = rowselect_cap(k);
  TFRS_DYN_SMEM(row_topk_kernel<AhProvider>, 64 * 1024);
  TFRS_DYN_SMEM(row_topk_kernel<RescoreProvider>, 64 * 1024);
  for (long long q0 = 0; q0 < Q; q0 += p.qc) {
    const int qc = (int)((Q - q0) < p.qc ? (Q - q0) : p.qc);
    const float* qq = q + q0 * d;
    int rc = tfrs_topk_scan_f32(qq, qc, centroids, L, d, P, 0, nullptr, nullptr, 0, probe_s, (int64_t*)probe_i, scan_ws,
                                p.scan, stream);
    if (rc) return rc;
    ta_lut<<<(unsigned)qc, 256, 0, st>>>(qq, d, codebooks, dpb, B, W, lut, scale);
    TFRS_LAUNCH_CHECK();
    const long long n_lists = (long long)P * p.S;
    AhProvider ah{lut, scale, probe_s, probe_i, leaf_offsets, codes, order, qc, P, p.S, W, kp, nullptr, 0, 0, 0.f, 0.f};
    row_topk_kernel<AhProvider><<<(unsigned)(n_lists * qc), RS_THREADS, rowselect_smem(cap_a, (size_t)W * 128), st>>>(
        ah, kp, cap_a, lists_s, lists_i, kp);
    TFRS_LAUNCH_CHECK();
    rc = tfrs_topk_merge_sorted_strided(lists_s, (const int64_t*)lists_i, (long long)qc * kp, (long long)qc * kp,
                                        (int)n_lists, qc, kp, kp, merged_s, (int64_t*)merged_i, stream);
    if (rc) return rc;
    const float* fs = merged_s;
    const long long* fi = merged_i;
    if (reorder) {
      RescoreProvider rp{qq, rows, merged_s, merged_i, d, kp};
      row_topk_kernel<RescoreProvider><<<(unsigned)qc, RS_THREADS, rowselect_smem(cap_r, 0), st>>>(rp, k, cap_r, resc_s,
                                                                                                    resc_i, k);
      TFRS_LAUNCH_CHECK();
      fs = resc_s; fi = resc_i;
    }
    ta_finalize<<<(unsigned)ceil_div((long long)qc * k, 256), 256, 0, st>>>(fs, fi, (long long)qc * k, out_scores + q0 * k,
                                                                            out_idx + q0 * k);
    TFRS_LAUNCH_CHECK();
  }
  return TFRS_OK;
}
