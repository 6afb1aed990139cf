// lookup.cu -- K15: the vocabulary hash tables of layers.StringLookup / layers.IntegerLookup (tf-keras index_lookup).
//
// Table: `cap` int32 slots (cap = a power of two >= 2V, at least 64), each holding a vocabulary position or -1, and for
// strings one 64-bit fingerprint per vocabulary entry.  The keys stay where the caller keeps them: the int64 vocabulary
// in order, or the vocabulary's bytes with int64 offsets.  Home slot: splitmix64's finalizer of an int64 key, SipHash-2-4
// (siphash.cuh, fixed key LK_K0 / LK_K1) of a string's bytes -- which is also its fingerprint -- masked to cap - 1;
// linear probing from there.
//
//   tfrs_lookup_build   one thread per vocabulary entry, atomicCAS on the slots; a probe that meets an equal key sets the
//                       duplicate flag.  Strings take one more launch before it for the fingerprints.  The slot layout
//                       may depend on the CAS race; a lookup's result never does.
//   tfrs_lookup         one thread per value, one launch: the mask test, then the probe (strings: fingerprint, then length,
//                       then bytes).  One int64 store per value; no atomics.  With a miss flag, a miss sets it.
//   tfrs_lookup_invert  one thread per index: a gather from the vocabulary, or a position code for strings.
//
// The table view and the string probe live in lookup.cuh, so that K16 (text.cu) probes the same tables the same way.
#include "lookup.cuh"

namespace tfrs {

constexpr int LK_THREADS = 256;
constexpr int64_t LK_MIN_SLOTS = 64;
constexpr int64_t LK_MAX_V = (1ll << 30) - 1;
constexpr uint64_t LK_K0 = 0x0706050403020100ull, LK_K1 = 0x0f0e0d0c0b0a0908ull;

__host__ __device__ __forceinline__ uint64_t lk_mix64(uint64_t z) {   // splitmix64's output function
  z += 0x9e3779b97f4a7c15ull;
  z = (z ^ (z >> 30)) * 0xbf58476d1ce4e5b9ull;
  z = (z ^ (z >> 27)) * 0x94d049bb133111ebull;
  return z ^ (z >> 31);
}

__device__ __forceinline__ uint64_t lk_fingerprint(const uint8_t* b, long long len) {
  return lk_fingerprint(b, len, LK_K0, LK_K1);
}

// ---- build ----------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(LK_THREADS) lk_build_i64_kernel(const LkTable t, int* __restrict__ dup) {
  const long long i = (long long)blockIdx.x * LK_THREADS + threadIdx.x;
  if (i >= t.V) return;
  const long long x = t.keys[i];
  unsigned long long s = lk_mix64((uint64_t)x) & t.cmask;
  for (;;) {
    const int cur = atomicCAS(t.slots + s, -1, (int)i);
    if (cur < 0) return;
    if (t.keys[cur] == x) { *dup = 1; return; }
    s = (s + 1) & t.cmask;
  }
}

__global__ void __launch_bounds__(LK_THREADS) lk_fingerprint_kernel(const LkTable t) {
  const long long i = (long long)blockIdx.x * LK_THREADS + threadIdx.x;
  if (i >= t.V) return;
  const long long o0 = t.offsets[i], o1 = t.offsets[i + 1];
  t.fp[i] = lk_fingerprint(t.bytes + o0, o1 - o0);
}

__global__ void __launch_bounds__(LK_THREADS) lk_build_bytes_kernel(const LkTable t, int* __restrict__ dup) {
  const long long i = (long long)blockIdx.x * LK_THREADS + threadIdx.x;
  if (i >= t.V) return;
  const unsigned long long h = t.fp[i];
  const long long o0 = t.offsets[i], len = t.offsets[i + 1] - o0;
  unsigned long long s = h & t.cmask;
  for (;;) {
    const int cur = atomicCAS(t.slots + s, -1, (int)i);
    if (cur < 0) return;
    if (t.fp[cur] == h) {
      const long long c0 = t.offsets[cur];
      if (t.offsets[cur + 1] - c0 == len && lk_bytes_equal(t.bytes + c0, t.bytes + o0, len)) { *dup = 1; return; }
    }
    s = (s + 1) & t.cmask;
  }
}

// ---- lookup ---------------------------------------------------------------------------------------------------------
// out = 0 for the mask, base + position for a vocabulary key; a miss gives oov, or -1 and sets *miss when miss != NULL.
template <typename T>
__global__ void __launch_bounds__(LK_THREADS)
lk_lookup_int_kernel(const LkTable t, const T* __restrict__ values, long long n, long long base, long long oov,
                     int* __restrict__ miss, long long* __restrict__ out) {
  const long long i = (long long)blockIdx.x * LK_THREADS + threadIdx.x;
  if (i >= n) return;
  const long long x = (long long)values[i];
  long long r = 0;
  if (!(t.has_mask && x == t.mask)) {
    const int* __restrict__ slots = t.slots;
    const long long* __restrict__ keys = t.keys;
    unsigned long long s = lk_mix64((uint64_t)x) & t.cmask;
    for (;;) {
      const int p = __ldg(slots + s);
      if (p < 0) {
        if (miss) { *miss = 1; r = -1; } else { r = oov; }
        break;
      }
      if (__ldg(keys + p) == x) { r = base + p; break; }
      s = (s + 1) & t.cmask;
    }
  }
  out[i] = r;
}

__global__ void __launch_bounds__(LK_THREADS)
lk_lookup_bytes_kernel(const LkTable t, const uint8_t* __restrict__ data, const long long* __restrict__ offsets,
                       long long n, long long base, long long oov, int* __restrict__ miss, long long* __restrict__ out) {
  const long long i = (long long)blockIdx.x * LK_THREADS + threadIdx.x;
  if (i >= n) return;
  const long long o0 = offsets[i], o1 = offsets[i + 1];
  const long long len = o1 > o0 ? o1 - o0 : 0;
  const uint8_t* b = data + o0;
  long long r = 0;
  if (!(t.has_mask && len == t.mask_len && lk_bytes_equal(b, t.mask_bytes, len))) {
    lk_probe_bytes(t, b, len, LK_K0, LK_K1, [&](int p) { r = base + p; }, [&] {
      if (miss) { *miss = 1; r = -1; } else { r = oov; }
    });
  }
  out[i] = r;
}

// ---- invert ---------------------------------------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(LK_THREADS)
lk_invert_kernel(const T* __restrict__ idx, long long n, const long long* __restrict__ keys, long long V, long long base,
                 int has_mask, long long mask_out, long long oov_out, long long* __restrict__ out) {
  const long long i = (long long)blockIdx.x * LK_THREADS + threadIdx.x;
  if (i >= n) return;
  const long long x = (long long)idx[i];
  long long r;
  if (x >= base && x - base < V) r = keys ? __ldg(keys + (x - base)) : x - base;
  else r = (has_mask && x == 0) ? mask_out : oov_out;
  out[i] = r;
}

static int64_t lk_slots(int64_t V) {
  int64_t cap = LK_MIN_SLOTS;
  while (cap < 2 * V) cap <<= 1;
  return cap;
}

static size_t lk_slot_bytes(int64_t V) { return align_up((size_t)lk_slots(V) * 4, 256); }

const uint64_t lk_string_key[2] = {LK_K0, LK_K1};

int lk_table(const tfrs_lookup_table* d, LkTable* t, const char* what) {
  TFRS_CHECK_ARG(d, "%s: NULL table", what);
  TFRS_CHECK_ARG(d->V >= 0 && d->V <= LK_MAX_V, "%s: V = %lld, must be in [0, 2^30)", what, (long long)d->V);
  TFRS_CHECK_ARG(d->kind == TFRS_I64 || d->kind == TFRS_BYTES, "%s: table kind must be I64 or BYTES", what);
  TFRS_CHECK_ARG(d->slots && ((uintptr_t)d->slots & 255) == 0, "%s: NULL or unaligned slots", what);
  // string bytes may be NULL when every key is empty (a zero-byte buffer)
  TFRS_CHECK_ARG(d->V == 0 || d->kind == TFRS_BYTES || d->keys, "%s: NULL keys", what);
  TFRS_CHECK_ARG(d->kind == TFRS_I64 || d->offsets, "%s: BYTES keys need offsets", what);
  TFRS_CHECK_ARG(!(d->kind == TFRS_BYTES && d->has_mask) || d->mask_len == 0 || d->mask_bytes,
                 "%s: NULL mask bytes", what);
  *t = LkTable{};
  t->slots = reinterpret_cast<int*>(d->slots);
  t->cmask = (unsigned long long)lk_slots(d->V) - 1;
  t->V = d->V;
  t->has_mask = d->has_mask ? 1 : 0;
  t->mask = d->mask;
  if (d->kind == TFRS_I64) {
    t->keys = reinterpret_cast<const long long*>(d->keys);
  } else {
    t->bytes = reinterpret_cast<const uint8_t*>(d->keys);
    t->offsets = reinterpret_cast<const long long*>(d->offsets);
    t->fp = reinterpret_cast<unsigned long long*>(reinterpret_cast<unsigned char*>(d->slots) + lk_slot_bytes(d->V));
    t->mask_bytes = d->mask_bytes;
    t->mask_len = d->mask_len;
  }
  return TFRS_OK;
}

}  // namespace tfrs

using namespace tfrs;

extern "C" int64_t tfrs_lookup_slots(int64_t V) { return V < 0 || V > LK_MAX_V ? -1 : lk_slots(V); }

extern "C" size_t tfrs_lookup_table_bytes(int64_t V, int kind) {
  if (V < 0 || V > LK_MAX_V || (kind != TFRS_I64 && kind != TFRS_BYTES)) return 0;
  return lk_slot_bytes(V) + (kind == TFRS_BYTES ? align_up((size_t)V * 8, 256) : 0);
}

extern "C" int tfrs_lookup_build(const tfrs_lookup_table* table, int32_t* dup, void* stream) {
  LkTable t;
  const int rc = lk_table(table, &t, "lookup_build");
  if (rc != TFRS_OK) return rc;
  TFRS_CHECK_ARG(dup, "lookup_build: NULL duplicate flag");
  cudaStream_t st = (cudaStream_t)stream;
  TFRS_CUDA(cudaMemsetAsync(t.slots, 0xff, (size_t)(t.cmask + 1) * 4, st));
  TFRS_CUDA(cudaMemsetAsync(dup, 0, 4, st));
  if (t.V == 0) return TFRS_OK;
  const unsigned grid = (unsigned)ceil_div(t.V, LK_THREADS);
  if (table->kind == TFRS_I64) {
    lk_build_i64_kernel<<<grid, LK_THREADS, 0, st>>>(t, dup);
    TFRS_LAUNCH_CHECK();
  } else {
    lk_fingerprint_kernel<<<grid, LK_THREADS, 0, st>>>(t);
    TFRS_LAUNCH_CHECK();
    lk_build_bytes_kernel<<<grid, LK_THREADS, 0, st>>>(t, dup);
    TFRS_LAUNCH_CHECK();
  }
  return TFRS_OK;
}

extern "C" int tfrs_lookup(const tfrs_lookup_table* table, const void* values, const int64_t* offsets, int kind, int64_t n,
                           int64_t base, int64_t oov, int32_t* miss, int64_t* out, void* stream) {
  LkTable t;
  const int rc = lk_table(table, &t, "lookup");
  if (rc != TFRS_OK) return rc;
  TFRS_CHECK_ARG(n >= 0 && n < (1ll << 38), "lookup: bad n = %lld", (long long)n);
  if (table->kind == TFRS_I64)
    TFRS_CHECK_ARG(kind == TFRS_I32 || kind == TFRS_I64, "lookup: an integer table takes I32 or I64 values");
  else
    TFRS_CHECK_ARG(kind == TFRS_BYTES, "lookup: a string table takes BYTES values");
  if (n == 0) return TFRS_OK;
  TFRS_CHECK_ARG(out && (kind == TFRS_BYTES ? offsets != nullptr : values != nullptr), "lookup: NULL values, offsets or out");
  cudaStream_t st = (cudaStream_t)stream;
  const unsigned grid = (unsigned)ceil_div(n, LK_THREADS);
  long long* o = reinterpret_cast<long long*>(out);
  if (kind == TFRS_I32)
    lk_lookup_int_kernel<int32_t><<<grid, LK_THREADS, 0, st>>>(t, (const int32_t*)values, n, base, oov, miss, o);
  else if (kind == TFRS_I64)
    lk_lookup_int_kernel<long long><<<grid, LK_THREADS, 0, st>>>(t, (const long long*)values, n, base, oov, miss, o);
  else
    lk_lookup_bytes_kernel<<<grid, LK_THREADS, 0, st>>>(t, (const uint8_t*)values, (const long long*)offsets, n, base, oov,
                                                        miss, o);
  TFRS_LAUNCH_CHECK();
  return TFRS_OK;
}

extern "C" int tfrs_lookup_invert(const void* idx, int kind, int64_t n, const int64_t* keys, int64_t V, int64_t base,
                                  int has_mask, int64_t mask_out, int64_t oov_out, int64_t* out, void* stream) {
  TFRS_CHECK_ARG(kind == TFRS_I32 || kind == TFRS_I64, "lookup_invert: indices must be I32 or I64");
  TFRS_CHECK_ARG(n >= 0 && n < (1ll << 38) && V >= 0 && V <= LK_MAX_V && base >= 0, "lookup_invert: bad n, V or base");
  if (n == 0) return TFRS_OK;
  TFRS_CHECK_ARG(idx && out, "lookup_invert: NULL idx or out");
  cudaStream_t st = (cudaStream_t)stream;
  const unsigned grid = (unsigned)ceil_div(n, LK_THREADS);
  const long long* k = reinterpret_cast<const long long*>(keys);
  long long* o = reinterpret_cast<long long*>(out);
  if (kind == TFRS_I32)
    lk_invert_kernel<int32_t><<<grid, LK_THREADS, 0, st>>>((const int32_t*)idx, n, k, V, base, has_mask, mask_out, oov_out, o);
  else
    lk_invert_kernel<long long><<<grid, LK_THREADS, 0, st>>>((const long long*)idx, n, k, V, base, has_mask, mask_out,
                                                             oov_out, o);
  TFRS_LAUNCH_CHECK();
  return TFRS_OK;
}
