// text.cu -- K16: layers.TextVectorization (tf-keras text_vectorization, output_mode="int", split="whitespace").
//
// Standardize: tf.strings.lower (ASCII only: bytes >= 0x80 are left alone), then Keras's DEFAULT_STRIP_REGEX, which
// deletes each of the 32 bytes of Python's string.punctuation.  Split: runs of the six ASCII whitespace bytes separate
// tokens; empty tokens are dropped.  A token's index comes from the K15 table of the layer's inner StringLookup
// (lookup.cuh's probe, on the same tables as lookup.cu).
//
//   tfrs_text_standardize  one thread per string: writes the standardized bytes into scratch at the string's own offsets
//                          (they are never longer than the input), fills the rest of its range with spaces, and counts
//                          its tokens (an atomicMax gives the longest count).
//   tfrs_text_lookup       one thread per string: walks its tokens in the scratch copy, probes the table for each, writes
//                          out[i, j] and the zero padding.  No atomics.
//   tfrs_text_spans        the same walk, writing each token's (offset, length) instead (adapt).
#include "lookup.cuh"

namespace tfrs {

constexpr int TX_THREADS = 256;

// Python's string.punctuation: !"#$%&'()*+,-./:;<=>?@[\]^_`{|}~
constexpr uint8_t TX_PUNCT[32] = {0x21, 0x22, 0x23, 0x24, 0x25, 0x26, 0x27, 0x28, 0x29, 0x2a, 0x2b, 0x2c, 0x2d, 0x2e, 0x2f,
                                  0x3a, 0x3b, 0x3c, 0x3d, 0x3e, 0x3f, 0x40, 0x5b, 0x5c, 0x5d, 0x5e, 0x5f, 0x60, 0x7b, 0x7c,
                                  0x7d, 0x7e};
// absl ascii_isspace: " \t\n\v\f\r"
constexpr uint8_t TX_SPACE[6] = {0x20, 0x09, 0x0a, 0x0b, 0x0c, 0x0d};

// bit (c - 64 * half) of the set's 64-bit word for bytes [64 * half, 64 * half + 64)
template <int N>
constexpr uint64_t tx_bits(const uint8_t (&set)[N], int half) {
  uint64_t w = 0;
  for (int k = 0; k < N; ++k)
    if (set[k] >> 6 == half) w |= 1ull << (set[k] & 63);
  return w;
}

constexpr uint64_t TX_PUNCT_LO = tx_bits(TX_PUNCT, 0), TX_PUNCT_HI = tx_bits(TX_PUNCT, 1);
constexpr uint64_t TX_SPACE_LO = tx_bits(TX_SPACE, 0);
static_assert(tx_bits(TX_SPACE, 1) == 0, "tx_space tests the low word only");

__device__ __forceinline__ bool tx_punct(uint32_t c) {
  return c < 128 && ((c < 64 ? TX_PUNCT_LO >> c : TX_PUNCT_HI >> (c - 64)) & 1);
}

__device__ __forceinline__ bool tx_space(uint32_t c) { return c < 64 && ((TX_SPACE_LO >> c) & 1); }

__global__ void __launch_bounds__(TX_THREADS)
tx_standardize_kernel(const uint8_t* __restrict__ data, const long long* __restrict__ offsets, long long n, int flags,
                      uint8_t* __restrict__ scratch, int* __restrict__ counts, int* __restrict__ max_count) {
  const long long i = (long long)blockIdx.x * TX_THREADS + threadIdx.x;
  if (i >= n) return;
  const long long o0 = offsets[i], o1 = offsets[i + 1];
  const bool lower = flags & TFRS_TEXT_LOWER, strip = flags & TFRS_TEXT_STRIP;
  long long w = o0;
  int count = 0;
  bool prev_space = true;
  for (long long k = o0; k < o1; ++k) {
    uint32_t c = data[k];
    if (lower && c - 'A' < 26u) c += 'a' - 'A';
    if (strip && tx_punct(c)) continue;
    const bool sp = tx_space(c);
    count += !sp && prev_space;
    prev_space = sp;
    scratch[w++] = (uint8_t)c;
  }
  for (; w < o1; ++w) scratch[w] = ' ';
  counts[i] = count;
  if (max_count && count) atomicMax(max_count, count);
}

// Walks the tokens of string i in the standardized copy; tok(j, start, len) for each until it returns false.
template <typename Tok>
__device__ __forceinline__ int tx_tokens(const uint8_t* __restrict__ s, long long o0, long long o1, Tok tok) {
  int j = 0;
  long long k = o0;
  for (;;) {
    while (k < o1 && tx_space(s[k])) ++k;
    if (k == o1) break;
    const long long start = k;
    while (k < o1 && !tx_space(s[k])) ++k;
    if (!tok(j, start, k - start)) break;
    ++j;
  }
  return j;
}

__global__ void __launch_bounds__(TX_THREADS)
tx_lookup_kernel(const LkTable t, uint64_t k0, uint64_t k1, const uint8_t* __restrict__ scratch,
                 const long long* __restrict__ offsets, long long n, long long T, long long base, long long oov,
                 long long* __restrict__ out) {
  const long long i = (long long)blockIdx.x * TX_THREADS + threadIdx.x;
  if (i >= n) return;
  long long* row = out + i * T;
  long long j = tx_tokens(scratch, offsets[i], offsets[i + 1], [&](int j, long long start, long long len) {
    if (j >= T) return false;
    long long r = oov;
    lk_probe_bytes(t, scratch + start, len, k0, k1, [&](int p) { r = base + p; }, [] {});
    row[j] = r;
    return true;
  });
  for (; j < T; ++j) row[j] = 0;
}

__global__ void __launch_bounds__(TX_THREADS)
tx_spans_kernel(const uint8_t* __restrict__ scratch, const long long* __restrict__ offsets, long long n,
                const long long* __restrict__ token_offsets, long long* __restrict__ spans) {
  const long long i = (long long)blockIdx.x * TX_THREADS + threadIdx.x;
  if (i >= n) return;
  long long* sp = spans + 2 * token_offsets[i];
  tx_tokens(scratch, offsets[i], offsets[i + 1], [&](int j, long long start, long long len) {
    sp[2 * j] = start;
    sp[2 * j + 1] = len;
    return true;
  });
}

}  // namespace tfrs

using namespace tfrs;

extern "C" int tfrs_text_standardize(const uint8_t* data, const int64_t* offsets, int64_t n, int64_t nbytes, int flags,
                                     uint8_t* scratch, int32_t* counts, int32_t* max_count, void* stream) {
  TFRS_CHECK_ARG(n >= 0 && n < (1ll << 31), "text_standardize: bad n = %lld", (long long)n);
  TFRS_CHECK_ARG(nbytes >= 0 && nbytes < (1ll << 32), "text_standardize: %lld bytes; at most 2^32 - 1",
                 (long long)nbytes);
  TFRS_CHECK_ARG((flags & ~(TFRS_TEXT_LOWER | TFRS_TEXT_STRIP)) == 0, "text_standardize: unknown flags %d", flags);
  cudaStream_t st = (cudaStream_t)stream;
  if (max_count) TFRS_CUDA(cudaMemsetAsync(max_count, 0, 4, st));
  if (n == 0) return TFRS_OK;
  TFRS_CHECK_ARG(offsets && counts && (nbytes == 0 || (data && scratch)), "text_standardize: NULL data, offsets, "
                 "scratch or counts");
  tx_standardize_kernel<<<(unsigned)ceil_div(n, TX_THREADS), TX_THREADS, 0, st>>>(
      data, reinterpret_cast<const long long*>(offsets), n, flags, scratch, counts, max_count);
  TFRS_LAUNCH_CHECK();
  return TFRS_OK;
}

extern "C" int tfrs_text_lookup(const tfrs_lookup_table* table, const uint8_t* scratch, const int64_t* offsets, int64_t n,
                                int64_t T, int64_t base, int64_t oov, int64_t* out, void* stream) {
  LkTable t;
  const int rc = lk_table(table, &t, "text_lookup");
  if (rc != TFRS_OK) return rc;
  TFRS_CHECK_ARG(table->kind == TFRS_BYTES, "text_lookup: the table must be a string (BYTES) table");
  TFRS_CHECK_ARG(n >= 0 && n < (1ll << 31) && T >= 0 && T < (1ll << 31) && n * T < (1ll << 40),
                 "text_lookup: bad n = %lld or T = %lld", (long long)n, (long long)T);
  if (n == 0 || T == 0) return TFRS_OK;
  TFRS_CHECK_ARG(offsets && out, "text_lookup: NULL offsets or out");
  tx_lookup_kernel<<<(unsigned)ceil_div(n, TX_THREADS), TX_THREADS, 0, (cudaStream_t)stream>>>(
      t, lk_string_key[0], lk_string_key[1], scratch, reinterpret_cast<const long long*>(offsets), n, T, base, oov,
      reinterpret_cast<long long*>(out));
  TFRS_LAUNCH_CHECK();
  return TFRS_OK;
}

extern "C" int tfrs_text_spans(const uint8_t* scratch, const int64_t* offsets, int64_t n, const int64_t* token_offsets,
                               int64_t* spans, void* stream) {
  TFRS_CHECK_ARG(n >= 0 && n < (1ll << 31), "text_spans: bad n = %lld", (long long)n);
  if (n == 0) return TFRS_OK;
  TFRS_CHECK_ARG(offsets && token_offsets, "text_spans: NULL offsets or token offsets");
  tx_spans_kernel<<<(unsigned)ceil_div(n, TX_THREADS), TX_THREADS, 0, (cudaStream_t)stream>>>(
      scratch, reinterpret_cast<const long long*>(offsets), n, reinterpret_cast<const long long*>(token_offsets),
      reinterpret_cast<long long*>(spans));
  TFRS_LAUNCH_CHECK();
  return TFRS_OK;
}
