/* unified_oracle.c -- plain C restatement of the UnifiedEmbedding hot path, the bar of the K8 kernels
 * (recommenders_b200/csrc/unified_embedding.cu).  Test infrastructure: built by tests/unified_oracle.py.
 *
 *  - SipHash-2-4 as in the SipHash paper (Aumasson & Bernstein, 2012), key (k0, k1) = the little-endian halves of the
 *    16 key bytes; tf.strings.to_hash_bucket_strong(input, num_buckets, key) = SipHash(key, bytes) % num_buckets.
 *  - tf.as_string of an int64: printf("%lld").
 *  - lookup / pooled lookup / its backward: straight loops in value order; fp32 sums from +0.0f, then one IEEE division
 *    by the count (mean) or by sqrtf(count) (sqrtn).  Compiled without FMA contraction or fast-math.
 */
#include <math.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#define ROTL(x, b) (uint64_t)(((x) << (b)) | ((x) >> (64 - (b))))
#define SIPROUND                                                   \
  do {                                                             \
    v0 += v1; v1 = ROTL(v1, 13); v1 ^= v0; v0 = ROTL(v0, 32);      \
    v2 += v3; v3 = ROTL(v3, 16); v3 ^= v2;                         \
    v0 += v3; v3 = ROTL(v3, 21); v3 ^= v0;                         \
    v2 += v1; v1 = ROTL(v1, 17); v1 ^= v2; v2 = ROTL(v2, 32);      \
  } while (0)

uint64_t uo_siphash(uint64_t k0, uint64_t k1, const uint8_t* m, int64_t len) {
  uint64_t v0 = k0 ^ 0x736f6d6570736575ull, v1 = k1 ^ 0x646f72616e646f6dull;
  uint64_t v2 = k0 ^ 0x6c7967656e657261ull, v3 = k1 ^ 0x7465646279746573ull;
  int64_t full = len / 8 * 8;
  for (int64_t i = 0; i < full; i += 8) {
    uint64_t w = 0;
    for (int k = 7; k >= 0; --k) w = (w << 8) | m[i + k];
    v3 ^= w; SIPROUND; SIPROUND; v0 ^= w;
  }
  uint64_t b = ((uint64_t)len) << 56;
  for (int64_t k = len - 1; k >= full; --k) b |= (uint64_t)m[k] << (8 * (k - full));
  v3 ^= b; SIPROUND; SIPROUND; v0 ^= b;
  v2 ^= 0xff;
  SIPROUND; SIPROUND; SIPROUND; SIPROUND;
  return v0 ^ v1 ^ v2 ^ v3;
}

int uo_as_string(int64_t x, char* buf) { return snprintf(buf, 24, "%lld", (long long)x); }

void uo_hash_i64(const int64_t* v, int64_t n, uint64_t k0, uint64_t k1, uint64_t num_bins, int64_t* out) {
  char buf[24];
  for (int64_t i = 0; i < n; ++i) {
    int len = uo_as_string(v[i], buf);
    out[i] = (int64_t)(uo_siphash(k0, k1, (const uint8_t*)buf, len) % num_bins);
  }
}

void uo_hash_bytes(const uint8_t* bytes, const int64_t* off, int64_t n, uint64_t k0, uint64_t k1, uint64_t num_bins,
                   int64_t* out) {
  for (int64_t i = 0; i < n; ++i) out[i] = (int64_t)(uo_siphash(k0, k1, bytes + off[i], off[i + 1] - off[i]) % num_bins);
}

/* out[i * ld + col + j] = table[ids[i] * dim + j] */
void uo_gather(const float* table, int dim, const int64_t* ids, int64_t n, float* out, int64_t ld, int64_t col) {
  for (int64_t i = 0; i < n; ++i) memcpy(out + i * ld + col, table + ids[i] * dim, sizeof(float) * dim);
}

static float uo_div(int combiner, int64_t count) { return combiner == 1 ? (float)count : sqrtf((float)count); }

/* combiner 0 sum, 1 mean, 2 sqrtn */
void uo_pool(const float* table, int dim, const int64_t* ids, const int64_t* splits, int64_t n_bags, int combiner,
             float* out, int64_t ld, int64_t col) {
  for (int64_t b = 0; b < n_bags; ++b) {
    const int64_t count = splits[b + 1] - splits[b];
    for (int j = 0; j < dim; ++j) {
      float acc = 0.0f;
      for (int64_t v = splits[b]; v < splits[b + 1]; ++v) acc = acc + table[ids[v] * dim + j];
      if (combiner != 0 && count > 0) acc = acc / uo_div(combiner, count);
      out[b * ld + col + j] = acc;
    }
  }
}

/* rows[v * dim + j] = grad[bag(v) * ld + col + j], divided as in uo_pool */
void uo_pool_bwd(const float* grad, int64_t ld, int64_t col, int dim, const int64_t* splits, int64_t n_bags, int combiner,
                 float* rows) {
  for (int64_t b = 0; b < n_bags; ++b) {
    const int64_t count = splits[b + 1] - splits[b];
    for (int64_t v = splits[b]; v < splits[b + 1]; ++v)
      for (int j = 0; j < dim; ++j) {
        float g = grad[b * ld + col + j];
        rows[v * dim + j] = combiner != 0 ? g / uo_div(combiner, count) : g;
      }
  }
}
