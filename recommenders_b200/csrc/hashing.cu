// hashing.cu -- K18: the bins of tf-keras Hashing (hashing.py `_hash_values_to_bins`), one launch per call.
//
// h = FarmHash Fingerprint64(message) without a salt (tf.strings.to_hash_bucket_fast, farmhash.cuh), or SipHash-2-4
// keyed by the salt (to_hash_bucket_strong, siphash.cuh).  The message is the value's bytes, or for integer values the
// decimal text of tf.as_string (bucket.cuh).  bin = h mod num_bins in unsigned 64-bit arithmetic; with a mask value and
// num_bins > 1, bin 0 is reserved: 0 for a value equal to the mask (compared as int64, or bytewise), else
// 1 + h mod (num_bins - 1).
//
// One thread per value and one int64 store per value; the hash is a template parameter, so each kernel holds one hash.
// Strings start at any byte offset and are read with byte loads only.
#include "common.cuh"
#include "bucket.cuh"
#include "farmhash.cuh"

namespace tfrs {

constexpr int HS_THREADS = 256;

struct HsParams {
  const void* values;
  const int64_t* offsets;
  long long n;
  int kind;
  int has_mask;                          // a value equal to the mask gets bin 0 (only when a bin is reserved for it)
  unsigned long long k0, k1;             // the SipHash key of the salted kernel
  unsigned long long nbins, magic;       // the modulus (num_bins, or num_bins - 1 with a reserved mask bin)
  long long first;                       // the lowest hashed bin: 1 with a reserved mask bin, else 0
  long long mask;
  const uint8_t* mask_bytes;
  long long mask_len;
  long long* bins;
};

__device__ __forceinline__ bool bytes_equal(const uint8_t* a, long long na, const uint8_t* b, long long nb) {
  if (na != nb) return false;
  for (long long k = 0; k < na; ++k)
    if (__ldg(a + k) != __ldg(b + k)) return false;
  return true;
}

template <bool kSalted>
__global__ void __launch_bounds__(HS_THREADS)
hashing_kernel(const __grid_constant__ HsParams P) {
  const long long i = (long long)blockIdx.x * HS_THREADS + threadIdx.x;
  if (i >= P.n) return;
  uint64_t h;
  bool masked;
  if (P.kind != TFRS_BYTES) {
    const long long x = P.kind == TFRS_I32 ? (long long)reinterpret_cast<const int32_t*>(P.values)[i]
                                           : reinterpret_cast<const long long*>(P.values)[i];
    masked = P.has_mask && x == P.mask;
    const Msg m = decimal_msg(x);
    h = kSalted ? siphash(m, nullptr, P.k0, P.k1) : fingerprint64_short(farm::MsgSrc{m.w0, m.w1, m.w2}, m.len);
  } else {
    const long long o0 = P.offsets[i], o1 = P.offsets[i + 1];
    const long long len = o1 > o0 ? o1 - o0 : 0;
    const uint8_t* b = reinterpret_cast<const uint8_t*>(P.values) + o0;
    masked = P.has_mask && bytes_equal(b, len, P.mask_bytes, P.mask_len);
    if (kSalted) {
      Msg m;
      const uint8_t* p = nullptr;
      bytes_msg(m, b, len, &p);
      h = siphash(m, p, P.k0, P.k1);
    } else {
      h = fingerprint64(farm::ByteSrc{b}, (uint64_t)len);
    }
  }
  P.bins[i] = masked ? 0 : P.first + (long long)mod_magic(h, P.nbins, P.magic);
}

}  // namespace tfrs
using namespace tfrs;

extern "C" int tfrs_hashing(const void* values, const int64_t* offsets, int kind, int64_t n, const uint64_t* salt,
                            int64_t num_bins, int has_mask, int64_t mask, const uint8_t* mask_bytes, int64_t mask_len,
                            int64_t* bins, void* stream) {
  TFRS_CHECK_ARG(n == 0 || (bins && values), "hashing: NULL argument");      // an empty call may pass NULL buffers
  TFRS_CHECK_ARG(kind == TFRS_I32 || kind == TFRS_I64 || (kind == TFRS_BYTES && offsets),
                 "hashing: kind must be I32, I64 or BYTES (with offsets)");
  TFRS_CHECK_ARG(n >= 0 && n < (1ll << 38) && num_bins >= 1, "hashing: bad n / num_bins");
  TFRS_CHECK_ARG(!has_mask || kind != TFRS_BYTES || (mask_len >= 0 && (mask_bytes || mask_len == 0)),
                 "hashing: a string mask needs mask_len >= 0 bytes at mask_bytes");
  if (n == 0) return TFRS_OK;
  HsParams p{};
  p.values = values; p.offsets = offsets; p.n = n; p.kind = kind; p.bins = reinterpret_cast<long long*>(bins);
  const bool reserve = has_mask && num_bins > 1;          // tf-keras reserves no bin when num_bins == 1
  p.has_mask = reserve;
  p.mask = mask; p.mask_bytes = mask_bytes; p.mask_len = mask_len;
  p.nbins = (unsigned long long)(reserve ? num_bins - 1 : num_bins);
  p.magic = ~0ull / p.nbins;
  p.first = reserve ? 1 : 0;
  const dim3 grid((unsigned)ceil_div(n, HS_THREADS));
  cudaStream_t st = (cudaStream_t)stream;
  if (salt) {
    p.k0 = salt[0]; p.k1 = salt[1];
    hashing_kernel<true><<<grid, HS_THREADS, 0, st>>>(p);
  } else {
    hashing_kernel<false><<<grid, HS_THREADS, 0, st>>>(p);
  }
  TFRS_LAUNCH_CHECK();
  return TFRS_OK;
}

extern "C" int tfrs_hash_bins(const void* values, const int64_t* offsets, int kind, int64_t n, const uint64_t* salt,
                              int64_t num_bins, int64_t* bins, void* stream) {
  TFRS_CHECK_ARG(salt, "hash_bins: NULL salt");
  return tfrs_hashing(values, offsets, kind, n, salt, num_bins, 0, 0, nullptr, 0, bins, stream);
}
