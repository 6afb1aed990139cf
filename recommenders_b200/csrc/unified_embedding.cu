// unified_embedding.cu -- K8: salted feature hashing fused with the shared-table row gather of UnifiedEmbedding
// (layers/feature_multiplexing/unified_embedding.py:186-215 with tf-keras Hashing(num_bins, salt) in front of every
// chunk lookup).
//
// bin = SipHash-2-4(k0 = salt[0], k1 = salt[1], message) mod num_bins  (tf.strings.to_hash_bucket_strong).  The message
// is the value's bytes, or for integer values the decimal text of tf.as_string ('-' for negatives, no padding).
//
// Forward, one launch for every feature of a call: a warp owns 32 consecutive values of one feature (blockIdx.y).
// Each lane forms its value's message words ONCE (decimal conversion or byte loads) and keeps them in three registers;
// then, chunk by chunk, it runs that chunk's SipHash and the warp copies the 32 rows K1-style (bucket ids travel by
// shuffle, up to 8 independent 16-byte row loads per thread before the first store).  Bucket ids are also written
// (when the caller asks for them) into per-table buffers, which is all a pooled (ragged) slot does in this launch.
// Pooled slots then take one more launch: a group of dim/4 lanes per (bag, slot) sums the bag's rows in value order.
// Backward: one launch writes each table's gradient rows, contiguous, in the caller's order.  No float atomics.
// Bucket ids alone (tfrs_hash_bins) come from K18's hash-only kernel (hashing.cu).
#include "common.cuh"
#include "bucket.cuh"
#include "bags.cuh"

namespace tfrs {

constexpr int UE_THREADS = 256;
constexpr int UE_MAX_FEATURES = 64;     // per launch; longer calls are split into groups (ue_groups)
constexpr int UE_MAX_SLOTS = 256;

struct UeFeat {
  const void* values;
  const int64_t* offsets;
  const int64_t* splits;
  long long n, n_bags;
  int first, n_chunks, kind, combiner;
  int copy;              // the forward kernel copies rows (unpooled); otherwise it only writes the bucket ids
};

struct UeSlot {
  const float* table;
  float* out;            // fwd: output; bwd: gradient rows out
  const float* grad;     // bwd: gradient of the output (same ld / col_off as the forward output)
  long long* ids;
  unsigned long long k0, k1, nbins, magic;
  long long ld;
  int col_off, dim;
};

struct UeParams {
  UeFeat f[UE_MAX_FEATURES];
  UeSlot s[UE_MAX_SLOTS];
  short y_slot[UE_MAX_SLOTS];      // pooling and backward launches: blockIdx.y -> slot, feature
  short y_feat[UE_MAX_SLOTS];
};
static_assert(sizeof(UeParams) <= 32000, "kernel parameters must stay under the 32 KB limit");

// The message of value i of a feature (kind: TFRS_I32, TFRS_I64, TFRS_BYTES); *p is the start of a byte string.
__device__ __forceinline__ Msg form_msg(const UeFeat& f, long long i, const uint8_t** p) {
  *p = nullptr;
  if (f.kind == TFRS_I32) return decimal_msg((long long)reinterpret_cast<const int32_t*>(f.values)[i]);
  if (f.kind == TFRS_I64) return decimal_msg(reinterpret_cast<const long long*>(f.values)[i]);
  const long long o0 = f.offsets[i], o1 = f.offsets[i + 1];
  const uint8_t* b = reinterpret_cast<const uint8_t*>(f.values) + o0;
  Msg m;
  bytes_msg(m, b, o1 > o0 ? o1 - o0 : 0, p);
  return m;
}

__global__ void __launch_bounds__(UE_THREADS)
ue_lookup_fwd_kernel(const __grid_constant__ UeParams P) {
  const UeFeat& f = P.f[blockIdx.y];
  const int lane = threadIdx.x & 31;
  const long long i0 = ((long long)blockIdx.x * (UE_THREADS / 32) + (threadIdx.x >> 5)) * 32;
  if (i0 >= f.n) return;                   // warp-uniform
  const long long i = i0 + lane;
  const bool valid = i < f.n;
  const uint8_t* p = nullptr;
  Msg m;
  if (valid) m = form_msg(f, i, &p);
  auto bin = [&](int c) -> long long {      // chunk c's bucket id of this lane's value (also stored when asked for)
    const UeSlot& s = P.s[f.first + c];
    long long r = 0;
    if (valid) {
      r = (long long)mod_magic(siphash(m, p, s.k0, s.k1), s.nbins, s.magic);
      if (s.ids) s.ids[i] = r;
    }
    return r;
  };
  if (!f.copy) {
    for (int c = 0; c < f.n_chunks; ++c) bin(c);
    return;
  }
  // chunk c's rows are copied while chunk c+1 is hashed: its SipHash runs between the first loads and their stores
  long long r = bin(0);
  for (int c = 0; c < f.n_chunks; ++c) {
    const UeSlot& s = P.s[f.first + c];
    long long r_next = 0;
    // warp-chunk row copy (K1): 32 rows of L float4 lanes, 32*L items, 8 items per lane in flight
    const float4* __restrict__ table = reinterpret_cast<const float4*>(s.table);
    float4* __restrict__ o4 = reinterpret_cast<float4*>(s.out + s.col_off);
    const int L = s.dim >> 2;
    const bool pow2 = (L & (L - 1)) == 0;
    const int lshift = 31 - __clz(L);
    const long long ld4 = s.ld >> 2;
    for (int s0 = 0; s0 < L; s0 += 8) {
      float4 v[8]; int jj[8];
#pragma unroll
      for (int u = 0; u < 8; ++u) {
        const int item = (s0 + u) * 32 + lane;
        const int j = pow2 ? item >> lshift : item / L;
        const int sub = item - j * L;
        const long long row = __shfl_sync(0xffffffffu, r, j & 31);
        jj[u] = (s0 + u < L && i0 + j < f.n) ? j : -1;
        v[u] = jj[u] >= 0 ? __ldg(table + row * L + sub) : make_float4(0.f, 0.f, 0.f, 0.f);
      }
      if (s0 == 0 && c + 1 < f.n_chunks) r_next = bin(c + 1);
#pragma unroll
      for (int u = 0; u < 8; ++u) {
        if (jj[u] >= 0) {
          const int item = (s0 + u) * 32 + lane;
          o4[(i0 + jj[u]) * ld4 + (item - jj[u] * L)] = v[u];
        }
      }
    }
    r = r_next;
  }
}

// combiner: 0 sum, 1 mean, 2 sqrtn (one IEEE division by count or by sqrtf(count); empty bags give zeros)
__device__ __forceinline__ float4 combine(float4 a, int combiner, long long count) {
  if (combiner == 0 || count == 0) return a;
  const float d = combiner == 1 ? (float)count : __fsqrt_rn((float)count);
  return make_float4(__fdiv_rn(a.x, d), __fdiv_rn(a.y, d), __fdiv_rn(a.z, d), __fdiv_rn(a.w, d));
}

// A group of dim/4 lanes per (bag, slot): the bag's rows summed in value order from +0, then the combiner.
__global__ void __launch_bounds__(UE_THREADS)
ue_pool_kernel(const __grid_constant__ UeParams P) {
  const UeSlot& s = P.s[P.y_slot[blockIdx.y]];
  const UeFeat& f = P.f[P.y_feat[blockIdx.y]];
  const int L = s.dim >> 2;
  const long long t = (long long)blockIdx.x * UE_THREADS + threadIdx.x;
  const long long b = t / L;
  if (b >= f.n_bags) return;
  const int sub = (int)(t - b * L);
  long long v0, v1;
  bag_range(f, b, &v0, &v1);
  const float4* __restrict__ table = reinterpret_cast<const float4*>(s.table);
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll 4
  for (long long v = v0; v < v1; ++v) {
    const float4 x = __ldg(table + s.ids[v] * L + sub);
    acc.x = __fadd_rn(acc.x, x.x); acc.y = __fadd_rn(acc.y, x.y);
    acc.z = __fadd_rn(acc.z, x.z); acc.w = __fadd_rn(acc.w, x.w);
  }
  reinterpret_cast<float4*>(s.out + s.col_off)[b * (s.ld >> 2) + sub] = combine(acc, f.combiner, v1 - v0);
}

// Backward: rows[v] = grad[v] (unpooled) or grad[bag(v)] scaled by the combiner (pooled; a value outside every bag gets
// a zero row).  blockIdx.y = slot; a grid-stride loop over the slot's n * dim/4 float4 items, 4 in flight per thread.
constexpr int UE_BWD_ITEMS = 4;

__global__ void __launch_bounds__(UE_THREADS)
ue_lookup_bwd_kernel(const __grid_constant__ UeParams P) {
  const UeSlot& s = P.s[P.y_slot[blockIdx.y]];
  const UeFeat& f = P.f[P.y_feat[blockIdx.y]];
  const int L = s.dim >> 2;
  const int lshift = (L & (L - 1)) == 0 ? 31 - __clz(L) : -1;
  const long long total = f.n * L, ld4 = s.ld >> 2;
  const long long stride = (long long)gridDim.x * UE_THREADS;
  // g4 is read with __ldg: beside bags.cuh's __ldg loads of the splits the compiler no longer picks the read-only path
  const float4* __restrict__ g4 = reinterpret_cast<const float4*>(s.grad + s.col_off);
  float4* __restrict__ rows = reinterpret_cast<float4*>(s.out);
  const bool pooled = f.splits != nullptr;
  for (long long e = (long long)blockIdx.x * UE_THREADS + threadIdx.x; e < total; e += stride * UE_BWD_ITEMS) {
    float4 v[UE_BWD_ITEMS];
#pragma unroll
    for (int u = 0; u < UE_BWD_ITEMS; ++u) {
      const long long w = e + u * stride;
      if (w >= total) break;
      const long long i = lshift >= 0 ? w >> lshift : w / L;
      const int sub = (int)(w - i * L);
      if (!pooled) { v[u] = __ldg(g4 + i * ld4 + sub); continue; }
      const long long lo = bag_of(f, i);
      long long a, z;
      bag_range(f, lo, &a, &z);
      v[u] = (i >= a && i < z) ? combine(__ldg(g4 + lo * ld4 + sub), f.combiner, z - a)
                               : make_float4(0.f, 0.f, 0.f, 0.f);
    }
#pragma unroll
    for (int u = 0; u < UE_BWD_ITEMS; ++u) {
      const long long w = e + u * stride;
      if (w < total) rows[w] = v[u];
    }
  }
}


// ---------------------------------------------------------------------------------------------------------------------
// Host side: the caller's features and slots are validated once, then packed into one UeParams per group that fits the
// parameter block (one group for up to 64 features and 256 slots).
static int ue_check(const tfrs_ue_feature* features, int n_features, const tfrs_ue_slot* slots, int n_slots, bool bwd,
                    const char* what) {
  TFRS_CHECK_ARG(features && slots && n_features > 0 && n_slots > 0, "%s: NULL argument or empty call", what);
  int total = 0;
  for (int k = 0; k < n_features; ++k) {
    const tfrs_ue_feature& f = features[k];
    TFRS_CHECK_ARG(f.n_chunks > 0, "%s: feature %d: n_chunks must be positive", what, k);
    TFRS_CHECK_ARG(f.n >= 0 && f.n < (1ll << 38), "%s: feature %d: bad n", what, k);
    TFRS_CHECK_ARG(!f.row_splits || (f.n_bags >= 0 && f.combiner >= TFRS_COMBINER_SUM && f.combiner <= TFRS_COMBINER_SQRTN),
                   "%s: feature %d: bad n_bags / combiner", what, k);
    // the backward finds a value's bag among bags 0 .. n_bags-1: pooled values need at least one bag
    TFRS_CHECK_ARG(!f.row_splits || f.n_bags >= 1 || f.n == 0, "%s: feature %d: %lld pooled values but no bag", what, k,
                   (long long)f.n);
    // rows of the forward output: an empty batch may come with NULL output / gradient pointers
    const long long out_rows = f.row_splits ? f.n_bags : f.n;
    if (!bwd)
      TFRS_CHECK_ARG(f.n == 0 || (f.values && (f.kind == TFRS_I32 || f.kind == TFRS_I64 || (f.kind == TFRS_BYTES && f.offsets))),
                     "%s: feature %d: NULL values, or kind not I32, I64 or BYTES with offsets", what, k);
    TFRS_CHECK_ARG(f.n_chunks <= n_slots - total, "%s: the features have more chunks than the %d slots", what, n_slots);
    for (int c = total; c < total + f.n_chunks; ++c) {
      const tfrs_ue_slot& s = slots[c];
      TFRS_CHECK_ARG(s.dim > 0 && s.dim % 4 == 0 && s.col_off >= 0 && s.col_off % 4 == 0 && s.ld % 4 == 0 &&
                     (int64_t)s.col_off + s.dim <= s.ld, "%s: slot %d: dim, col_off and ld must be multiples of 4, "
                     "the columns inside ld", what, c);
      if (!bwd) {
        TFRS_CHECK_ARG(s.table && s.rows > 0 && (s.out || out_rows == 0) && ((uintptr_t)s.table & 15) == 0 &&
                       ((uintptr_t)s.out & 15) == 0, "%s: slot %d: NULL or unaligned table / out, or no rows", what, c);
        TFRS_CHECK_ARG(!f.row_splits || s.ids || f.n == 0, "%s: slot %d: a pooled slot needs its bucket-id buffer", what,
                       c);
      } else {
        TFRS_CHECK_ARG(((s.grad && s.grad_rows) || f.n == 0) && ((uintptr_t)s.grad & 15) == 0 &&
                       ((uintptr_t)s.grad_rows & 15) == 0,
                       "%s: slot %d: NULL or unaligned grad / grad_rows", what, c);
      }
    }
    total += f.n_chunks;
  }
  TFRS_CHECK_ARG(total == n_slots, "%s: the features have %d chunks, n_slots is %d", what, total, n_slots);
  return TFRS_OK;
}

// Calls launch(params, features in the group, slots in the group) once per group; y_slot / y_feat start as the identity
// map over the group's slots (the backward launch), the forward rewrites them for its pooling launch.  A feature goes
// whole into the current group, or into a fresh one when its chunks do not fit.  A feature of more than UE_MAX_SLOTS
// chunks fills the current group and continues in fresh ones, one UeFeat entry per group over a disjoint range of its
// chunks: every slot carries its own salt, table and columns, so the chunks of a feature are independent.
template <typename Launch>
static int ue_groups(const tfrs_ue_feature* features, int n_features, const tfrs_ue_slot* slots, bool bwd, Launch launch) {
  UeParams p;
  int nf = 0, ns = 0, slot0 = 0;
  for (int k = 0; k < n_features; ++k) {
    const tfrs_ue_feature& f = features[k];
    for (int c0 = 0; c0 < f.n_chunks;) {
      if (nf > 0 && (nf == UE_MAX_FEATURES || ns == UE_MAX_SLOTS ||
                     (f.n_chunks <= UE_MAX_SLOTS && ns + f.n_chunks > UE_MAX_SLOTS))) {
        const int rc = launch(p, nf, ns);
        if (rc != TFRS_OK) return rc;
        nf = 0; ns = 0;
      }
      const int nc = min(f.n_chunks - c0, UE_MAX_SLOTS - ns);
      UeFeat& d = p.f[nf];
      d.values = f.values; d.offsets = f.offsets; d.splits = f.row_splits; d.n = f.n;
      d.n_bags = f.row_splits ? f.n_bags : 0; d.first = ns; d.n_chunks = nc; d.kind = f.kind;
      d.combiner = f.combiner; d.copy = f.row_splits ? 0 : 1;
      for (int c = 0; c < nc; ++c) {
        const tfrs_ue_slot& s = slots[slot0 + c0 + c];
        UeSlot& o = p.s[ns + c];
        o.table = s.table; o.grad = s.grad; o.out = bwd ? s.grad_rows : s.out;
        o.ids = reinterpret_cast<long long*>(s.ids);
        o.k0 = s.salt[0]; o.k1 = s.salt[1];
        o.nbins = (unsigned long long)(s.rows > 0 ? s.rows : 1); o.magic = ~0ull / o.nbins;
        o.ld = s.ld; o.col_off = s.col_off; o.dim = s.dim;
        p.y_slot[ns + c] = (short)(ns + c); p.y_feat[ns + c] = (short)nf;
      }
      c0 += nc; ns += nc; ++nf;
    }
    slot0 += f.n_chunks;
  }
  return nf > 0 ? launch(p, nf, ns) : TFRS_OK;
}

}  // namespace tfrs
using namespace tfrs;

extern "C" int tfrs_unified_lookup_fwd_f32(const tfrs_ue_feature* features, int n_features, const tfrs_ue_slot* slots,
                                           int n_slots, void* stream) {
  const int rc = ue_check(features, n_features, slots, n_slots, false, "unified_lookup_fwd");
  if (rc != TFRS_OK) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  return ue_groups(features, n_features, slots, false, [&](UeParams& p, int nf, int) -> int {
    long long max_n = 0, max_pool = 0;
    int np = 0;
    for (int k = 0; k < nf; ++k) {
      max_n = max(max_n, p.f[k].n);
      if (p.f[k].copy) continue;
      for (int c = 0; c < p.f[k].n_chunks; ++c) {   // the pooling launch runs over the pooled slots only
        const int si = p.f[k].first + c;
        p.y_slot[np] = (short)si; p.y_feat[np] = (short)k; ++np;
        max_pool = max(max_pool, p.f[k].n_bags * (p.s[si].dim >> 2));
      }
    }
    if (max_n > 0) {
      ue_lookup_fwd_kernel<<<dim3((unsigned)ceil_div(max_n, UE_THREADS), (unsigned)nf), UE_THREADS, 0, st>>>(p);
      TFRS_LAUNCH_CHECK();
    }
    if (max_pool > 0) {
      ue_pool_kernel<<<dim3((unsigned)ceil_div(max_pool, UE_THREADS), (unsigned)np), UE_THREADS, 0, st>>>(p);
      TFRS_LAUNCH_CHECK();
    }
    return TFRS_OK;
  });
}

extern "C" int tfrs_unified_lookup_bwd_f32(const tfrs_ue_feature* features, int n_features, const tfrs_ue_slot* slots,
                                           int n_slots, void* stream) {
  const int rc = ue_check(features, n_features, slots, n_slots, true, "unified_lookup_bwd");
  if (rc != TFRS_OK) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  return ue_groups(features, n_features, slots, true, [&](UeParams& p, int nf, int ns) -> int {
    long long max_items = 0;
    for (int k = 0; k < nf; ++k)
      for (int c = 0; c < p.f[k].n_chunks; ++c) max_items = max(max_items, p.f[k].n * (p.s[p.f[k].first + c].dim >> 2));
    if (max_items == 0) return TFRS_OK;
    const long long want = ceil_div(max_items, (long long)UE_THREADS * UE_BWD_ITEMS);
    ue_lookup_bwd_kernel<<<dim3((unsigned)min(want, 1ll << 20), (unsigned)ns), UE_THREADS, 0, st>>>(p);
    TFRS_LAUNCH_CHECK();
    return TFRS_OK;
  });
}
