// embedding_bag.cu -- K11: weighted multi-hot bag pooling of TPUEmbedding (layers/embedding/tpu_embedding_layer.py, the
// TPUEmbeddingForServing path: tf.nn.safe_embedding_lookup_sparse per feature), every feature of a call in one launch.
//
// A feature reads one table [rows, dim] with n ids (I32 / I64) and optional fp32 weights [n], and is one of
//   pooled    (row_splits, max_seq_len == 0): out row b = (sum over the bag's valid values of w*e, in value order from
//             +0.0f, one __fmul_rn and one __fadd_rn per value) / D, D = 1 (sum), sum w (mean), sqrtf(sum w*w) (sqrtn),
//             D summed sequentially in fp32 in value order; one IEEE division (none for sum); an empty bag gives zeros.
//   sequence  (row_splits, max_seq_len L > 0): out row b*L + j = w_j * e_j for j < min(L, bag size), zeros elsewhere.
//   dense     (row_splits == NULL): out row i = e_i (no weights, no combiner).
// Ids outside [0, rows) are dropped with their weight: they add nothing to a bag or its denominator, and give a zero row
// (dense and sequence positions) and a zero gradient row.
// Forward: blockIdx.y = feature; a thread owns one 16-byte piece (dim % 4 == 0 and aligned) or one column of one output
//   row, so a group of dim/4 (or dim) consecutive threads covers a row.  A pooled bag is walked in batches of BG_BATCH
//   values: ids and weights first, then the BG_BATCH row loads in flight, then the in-order adds.  The same launch copies
//   the ids to the caller's int64 buffer (the backward pair's ids) and, for mean / sqrtn, writes each bag's D.
// Backward: one launch, blockIdx.y = feature, a grid-stride loop over the feature's (value, piece) items: a pooled value
//   finds its bag by binary search over row_splits and writes (g_b * w) / D_b (g_b * w for sum); a sequence value writes
//   g_{b,j} * w (zeros past L); a dense value writes g_i.  Every value writes its row: no float atomics.
// HBM bytes, forward: V*(id + weight) + V_valid*dim*4 (rows) + R*dim*4 (outputs) [+ V*8 ids, + bags*4 D];
//            backward: V*(id + weight) + V*dim*4 (rows written) + gradient rows read (each bag's gradient once per value,
//            mostly from L2).  V = values, R = output rows.
#include "common.cuh"
#include "bags.cuh"

namespace tfrs {

constexpr int BG_THREADS = 256;
constexpr int BG_MAX_FEATURES = 128;   // per launch; longer calls are split into groups of whole features
constexpr int BG_BATCH = 4;            // pooled: row loads in flight per thread
constexpr int BG_BWD_ITEMS = 4;

struct BagFeat {
  const float* table;
  const void* values;
  const int64_t* splits;       // NULL: dense
  const float* weights;        // NULL: all 1
  float* out;
  long long* ids;              // forward: nullable
  float* denom;                // forward: nullable (mean / sqrtn); backward: read
  const float* grad;           // backward
  float* grad_rows;            // backward
  long long rows, n, n_bags, ld;
  int dim, col_off, combiner, seq_len, kind, vec;
};

struct BagParams {
  BagFeat f[BG_MAX_FEATURES];
};
static_assert(sizeof(BagParams) <= 32000, "kernel parameters must stay under the 32 KB limit");

__device__ __forceinline__ long long bg_id(const BagFeat& f, long long v) {
  return f.kind == TFRS_I32 ? (long long)__ldg(reinterpret_cast<const int32_t*>(f.values) + v)
                            : __ldg(reinterpret_cast<const long long*>(f.values) + v);
}

__device__ __forceinline__ float bg_w(const BagFeat& f, long long v) { return f.weights ? __ldg(f.weights + v) : 1.f; }

// V = 4: float4 pieces; V = 1: single columns.  The arithmetic is per column and identical in both.
template <int V> struct Vec;
template <> struct Vec<4> {
  using T = float4;
  __device__ __forceinline__ static T zero() { return make_float4(0.f, 0.f, 0.f, 0.f); }
  __device__ __forceinline__ static T load(const float* p) { return __ldg(reinterpret_cast<const float4*>(p)); }
  __device__ __forceinline__ static void store(float* p, T x) { *reinterpret_cast<float4*>(p) = x; }
  __device__ __forceinline__ static T mul(T a, float s) {
    return make_float4(__fmul_rn(a.x, s), __fmul_rn(a.y, s), __fmul_rn(a.z, s), __fmul_rn(a.w, s));
  }
  __device__ __forceinline__ static T div(T a, float s) {
    return make_float4(__fdiv_rn(a.x, s), __fdiv_rn(a.y, s), __fdiv_rn(a.z, s), __fdiv_rn(a.w, s));
  }
  __device__ __forceinline__ static T axpy(T acc, float w, T e) {   // acc + w*e, two roundings per column
    return make_float4(__fadd_rn(acc.x, __fmul_rn(w, e.x)), __fadd_rn(acc.y, __fmul_rn(w, e.y)),
                       __fadd_rn(acc.z, __fmul_rn(w, e.z)), __fadd_rn(acc.w, __fmul_rn(w, e.w)));
  }
};
template <> struct Vec<1> {
  using T = float;
  __device__ __forceinline__ static T zero() { return 0.f; }
  __device__ __forceinline__ static T load(const float* p) { return __ldg(p); }
  __device__ __forceinline__ static void store(float* p, T x) { *p = x; }
  __device__ __forceinline__ static T mul(T a, float s) { return __fmul_rn(a, s); }
  __device__ __forceinline__ static T div(T a, float s) { return __fdiv_rn(a, s); }
  __device__ __forceinline__ static T axpy(T acc, float w, T e) { return __fadd_rn(acc, __fmul_rn(w, e)); }
};

// One output row piece: pooled bag b, sequence position (b, j), or dense value i.  `col` is the piece's first column.
template <int V>
__device__ __forceinline__ void bg_fwd_item(const BagFeat& f, long long r, int col) {
  using X = Vec<V>;
  typename X::T acc = X::zero();
  if (!f.splits) {                                            // dense
    const long long id = bg_id(f, r);
    if (id >= 0 && id < f.rows) acc = X::load(f.table + id * f.dim + col);
  } else if (f.seq_len > 0) {                                 // sequence
    const long long b = r / f.seq_len;
    const int j = (int)(r - b * f.seq_len);
    long long s0, s1;
    bag_range(f, b, &s0, &s1);
    if (s0 + j < s1) {
      const long long id = bg_id(f, s0 + j);
      if (id >= 0 && id < f.rows) acc = X::mul(X::load(f.table + id * f.dim + col), bg_w(f, s0 + j));
    }
  } else {                                                    // pooled
    long long s0, s1;
    bag_range(f, r, &s0, &s1);
    float den = 0.f;
    bool any = false;
    for (long long v0 = s0; v0 < s1; v0 += BG_BATCH) {
      long long id[BG_BATCH]; float w[BG_BATCH];
#pragma unroll
      for (int u = 0; u < BG_BATCH; ++u) {
        id[u] = v0 + u < s1 ? bg_id(f, v0 + u) : -1;
        w[u] = v0 + u < s1 ? bg_w(f, v0 + u) : 0.f;
        if (id[u] >= f.rows) id[u] = -1;
      }
      typename X::T e[BG_BATCH];
#pragma unroll
      for (int u = 0; u < BG_BATCH; ++u) e[u] = id[u] >= 0 ? X::load(f.table + id[u] * f.dim + col) : X::zero();
#pragma unroll
      for (int u = 0; u < BG_BATCH; ++u) {
        if (id[u] < 0) continue;
        any = true;
        acc = X::axpy(acc, w[u], e[u]);
        if (f.combiner == TFRS_COMBINER_MEAN) den = __fadd_rn(den, w[u]);
        else if (f.combiner == TFRS_COMBINER_SQRTN) den = __fadd_rn(den, __fmul_rn(w[u], w[u]));
      }
    }
    if (f.combiner != TFRS_COMBINER_SUM) {
      if (f.combiner == TFRS_COMBINER_SQRTN) den = __fsqrt_rn(den);
      if (any) acc = X::div(acc, den);
      if (f.denom && col == 0) f.denom[r] = den;
    }
  }
  X::store(f.out + r * f.ld + f.col_off + col, acc);
}

// The minimum of 4 blocks per SM is a register budget of 64: under ptxas's default choice (48) the calls of the IEEE
// division's slow path spill 12 bytes.
__global__ void __launch_bounds__(BG_THREADS, 4)
bg_fwd_kernel(const __grid_constant__ BagParams P) {
  const BagFeat& f = P.f[blockIdx.y];
  const long long t = (long long)blockIdx.x * BG_THREADS + threadIdx.x;
  const long long nthreads = (long long)gridDim.x * BG_THREADS;
  if (f.ids)
    for (long long v = t; v < f.n; v += nthreads) f.ids[v] = bg_id(f, v);
  const int P4 = f.vec ? f.dim >> 2 : f.dim;                 // pieces per row
  const long long out_rows = !f.splits ? f.n : (f.seq_len > 0 ? f.n_bags * f.seq_len : f.n_bags);
  for (long long e = t; e < out_rows * P4; e += nthreads) {
    const long long r = e / P4;
    const int p = (int)(e - r * P4);
    if (f.vec) bg_fwd_item<4>(f, r, p * 4);
    else bg_fwd_item<1>(f, r, p);
  }
}

template <int V>
__device__ __forceinline__ typename Vec<V>::T bg_bwd_item(const BagFeat& f, long long v, int col) {
  using X = Vec<V>;
  const long long id = bg_id(f, v);
  if (id < 0 || id >= f.rows) return X::zero();
  if (!f.splits) return X::load(f.grad + v * f.ld + f.col_off + col);
  const long long lo = bag_of(f, v);
  long long s0, s1;
  bag_range(f, lo, &s0, &s1);
  if (v < s0 || v >= s1) return X::zero();
  const float w = bg_w(f, v);
  if (f.seq_len > 0) {
    const long long j = v - s0;
    return j < f.seq_len ? X::mul(X::load(f.grad + (lo * f.seq_len + j) * f.ld + f.col_off + col), w) : X::zero();
  }
  const typename X::T g = X::mul(X::load(f.grad + lo * f.ld + f.col_off + col), w);
  return f.combiner == TFRS_COMBINER_SUM ? g : X::div(g, __ldg(f.denom + lo));
}

__global__ void __launch_bounds__(BG_THREADS)
bg_bwd_kernel(const __grid_constant__ BagParams P) {
  const BagFeat& f = P.f[blockIdx.y];
  const int P4 = f.vec ? f.dim >> 2 : f.dim;
  const long long total = f.n * P4;
  const long long stride = (long long)gridDim.x * BG_THREADS;
  for (long long e = (long long)blockIdx.x * BG_THREADS + threadIdx.x; e < total; e += stride * BG_BWD_ITEMS) {
    if (f.vec) {
      float4 x[BG_BWD_ITEMS];
#pragma unroll
      for (int u = 0; u < BG_BWD_ITEMS; ++u) {
        const long long w = e + u * stride;
        if (w >= total) break;
        const long long v = w / P4;
        x[u] = bg_bwd_item<4>(f, v, (int)(w - v * P4) * 4);
      }
#pragma unroll
      for (int u = 0; u < BG_BWD_ITEMS; ++u) {
        const long long w = e + u * stride;
        if (w < total) reinterpret_cast<float4*>(f.grad_rows)[w] = x[u];
      }
    } else {
      float x[BG_BWD_ITEMS];
#pragma unroll
      for (int u = 0; u < BG_BWD_ITEMS; ++u) {
        const long long w = e + u * stride;
        if (w >= total) break;
        const long long v = w / P4;
        x[u] = bg_bwd_item<1>(f, v, (int)(w - v * P4));
      }
#pragma unroll
      for (int u = 0; u < BG_BWD_ITEMS; ++u) {
        const long long w = e + u * stride;
        if (w < total) f.grad_rows[w] = x[u];
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// Host side.
static bool aligned16(const void* p) { return ((uintptr_t)p & 15) == 0; }

static long long bg_out_rows(const tfrs_bag_feature& f) {
  return !f.row_splits ? f.n : (f.max_seq_len > 0 ? f.n_bags * f.max_seq_len : f.n_bags);
}

static int bg_check(const tfrs_bag_feature* features, int n_features, bool bwd, const char* what) {
  TFRS_CHECK_ARG(features && n_features > 0, "%s: NULL argument or empty call", what);
  for (int k = 0; k < n_features; ++k) {
    const tfrs_bag_feature& f = features[k];
    TFRS_CHECK_ARG(f.dim > 0 && f.rows > 0 && f.table, "%s: feature %d: NULL table, or no rows or columns", what, k);
    TFRS_CHECK_ARG(f.kind == TFRS_I32 || f.kind == TFRS_I64, "%s: feature %d: kind must be I32 or I64", what, k);
    TFRS_CHECK_ARG(f.n >= 0 && f.n < (1ll << 40) && (f.n == 0 || f.values), "%s: feature %d: bad n / values", what, k);
    TFRS_CHECK_ARG(f.max_seq_len >= 0, "%s: feature %d: max_seq_len < 0", what, k);
    TFRS_CHECK_ARG(f.row_splits || (!f.weights && f.max_seq_len == 0),
                   "%s: feature %d: a dense feature takes no weights and no max_seq_len", what, k);
    TFRS_CHECK_ARG(!f.row_splits || (f.n_bags >= 0 && f.combiner >= TFRS_COMBINER_SUM && f.combiner <= TFRS_COMBINER_SQRTN),
                   "%s: feature %d: bad n_bags / combiner", what, k);
    // the backward finds a value's bag among bags 0 .. n_bags-1: bagged values need at least one bag
    TFRS_CHECK_ARG(!f.row_splits || f.n_bags >= 1 || f.n == 0, "%s: feature %d: %lld values but no bag", what, k,
                   (long long)f.n);
    TFRS_CHECK_ARG(f.col_off >= 0 && (int64_t)f.col_off + f.dim <= f.ld, "%s: feature %d: columns outside ld", what, k);
    const long long rows_out = bg_out_rows(f);
    if (!bwd) {
      TFRS_CHECK_ARG(f.out || rows_out == 0, "%s: feature %d: NULL out", what, k);
    } else {
      TFRS_CHECK_ARG(f.n == 0 || (f.grad && f.grad_rows), "%s: feature %d: NULL grad / grad_rows", what, k);
      TFRS_CHECK_ARG(f.n == 0 || !f.row_splits || f.max_seq_len > 0 || f.combiner == TFRS_COMBINER_SUM || f.denom,
                     "%s: feature %d: mean / sqrtn need the forward's denominators", what, k);
    }
  }
  return TFRS_OK;
}

// Packs groups of whole features (at most BG_MAX_FEATURES each) and calls launch(params, features in the group).
template <typename Launch>
static int bg_groups(const tfrs_bag_feature* features, int n_features, bool bwd, Launch launch) {
  BagParams p;
  for (int k0 = 0; k0 < n_features; k0 += BG_MAX_FEATURES) {
    const int nf = min(n_features - k0, BG_MAX_FEATURES);
    for (int k = 0; k < nf; ++k) {
      const tfrs_bag_feature& f = features[k0 + k];
      BagFeat& d = p.f[k];
      d.table = f.table; d.values = f.values; d.splits = f.row_splits; d.weights = f.weights;
      d.out = f.out; d.ids = reinterpret_cast<long long*>(f.ids); d.denom = f.denom;
      d.grad = f.grad; d.grad_rows = f.grad_rows;
      d.rows = f.rows; d.n = f.n; d.n_bags = f.row_splits ? f.n_bags : 0; d.ld = f.ld;
      d.dim = f.dim; d.col_off = f.col_off; d.combiner = f.combiner; d.seq_len = f.row_splits ? f.max_seq_len : 0;
      d.kind = f.kind;
      const bool v = f.dim % 4 == 0 && f.col_off % 4 == 0 && f.ld % 4 == 0 && aligned16(f.table);
      d.vec = v && (bwd ? aligned16(f.grad) && aligned16(f.grad_rows) : aligned16(f.out));
    }
    const int rc = launch(p, nf);
    if (rc != TFRS_OK) return rc;
  }
  return TFRS_OK;
}

}  // namespace tfrs
using namespace tfrs;

extern "C" int tfrs_embedding_bag_fwd_f32(const tfrs_bag_feature* features, int n_features, void* stream) {
  const int rc = bg_check(features, n_features, false, "embedding_bag_fwd");
  if (rc != TFRS_OK) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  return bg_groups(features, n_features, false, [&](BagParams& p, int nf) -> int {
    long long items = 0;
    for (int k = 0; k < nf; ++k) {
      const BagFeat& f = p.f[k];
      const long long rows_out = !f.splits ? f.n : (f.seq_len > 0 ? f.n_bags * f.seq_len : f.n_bags);
      items = max(items, max(rows_out * (f.vec ? f.dim / 4 : f.dim), f.ids ? f.n : 0ll));
    }
    if (items == 0) return TFRS_OK;
    bg_fwd_kernel<<<dim3((unsigned)min((long long)ceil_div(items, BG_THREADS), 1ll << 24), (unsigned)nf), BG_THREADS, 0, st>>>(p);
    TFRS_LAUNCH_CHECK();
    return TFRS_OK;
  });
}

extern "C" int tfrs_embedding_bag_bwd_f32(const tfrs_bag_feature* features, int n_features, void* stream) {
  const int rc = bg_check(features, n_features, true, "embedding_bag_bwd");
  if (rc != TFRS_OK) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  return bg_groups(features, n_features, true, [&](BagParams& p, int nf) -> int {
    long long items = 0;
    for (int k = 0; k < nf; ++k) items = max(items, p.f[k].n * (p.f[k].vec ? p.f[k].dim / 4 : p.f[k].dim));
    if (items == 0) return TFRS_OK;
    const long long want = ceil_div(items, (long long)BG_THREADS * BG_BWD_ITEMS);
    bg_bwd_kernel<<<dim3((unsigned)min((long long)want, 1ll << 20), (unsigned)nf), BG_THREADS, 0, st>>>(p);
    TFRS_LAUNCH_CHECK();
    return TFRS_OK;
  });
}
