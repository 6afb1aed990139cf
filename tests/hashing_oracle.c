/* hashing_oracle.c -- plain C restatement of tf-keras Hashing, the bar of the K18 kernel (recommenders_b200/csrc/hashing.cu).
 * Test infrastructure: built by tests/hashing_oracle.py together with unified_oracle.c, whose SipHash-2-4 (uo_siphash)
 * and tf.as_string (uo_as_string) it calls.
 *
 *  - Fingerprint64 = farmhashna::Hash64 of the published FarmHash (tf.strings.to_hash_bucket_fast), byte by byte: every
 *    fetch is assembled from single bytes, little-endian.
 *  - hashing.py `_hash_values_to_bins`: h mod num_bins (unsigned); with a mask and num_bins > 1, 0 for the mask and
 *    1 + h mod (num_bins - 1) for every other value.
 */
#include <stdint.h>
#include <string.h>

uint64_t uo_siphash(uint64_t k0, uint64_t k1, const uint8_t* m, int64_t len);
int uo_as_string(int64_t x, char* buf);

static const uint64_t K0 = 0xc3a5c85c97cb3127ull, K1 = 0xb492b66fbe98f273ull, K2 = 0x9ae16a3b2f90404full;

static uint64_t fetch(const uint8_t* p, int n) {
  uint64_t v = 0;
  for (int k = n - 1; k >= 0; --k) v = (v << 8) | p[k];
  return v;
}
#define F64(p) fetch((p), 8)
#define F32(p) fetch((p), 4)

static uint64_t rot(uint64_t v, int s) { return s == 0 ? v : (v >> s) | (v << (64 - s)); }
static uint64_t smix(uint64_t v) { return v ^ (v >> 47); }

static uint64_t hl16(uint64_t u, uint64_t v, uint64_t mul) {
  uint64_t a = (u ^ v) * mul;
  a ^= a >> 47;
  uint64_t b = (v ^ a) * mul;
  b ^= b >> 47;
  return b * mul;
}

static uint64_t h0to16(const uint8_t* s, uint64_t len) {
  if (len >= 8) {
    uint64_t mul = K2 + len * 2, a = F64(s) + K2, b = F64(s + len - 8);
    uint64_t c = rot(b, 37) * mul + a, d = (rot(a, 25) + b) * mul;
    return hl16(c, d, mul);
  }
  if (len >= 4) {
    uint64_t mul = K2 + len * 2, a = F32(s);
    return hl16(len + (a << 3), F32(s + len - 4), mul);
  }
  if (len > 0) {
    uint32_t y = (uint32_t)s[0] + ((uint32_t)s[len >> 1] << 8);
    uint32_t z = (uint32_t)len + ((uint32_t)s[len - 1] << 2);
    return smix((uint64_t)y * K2 ^ (uint64_t)z * K0) * K2;
  }
  return K2;
}

static uint64_t h17to32(const uint8_t* s, uint64_t len) {
  uint64_t mul = K2 + len * 2;
  uint64_t a = F64(s) * K1, b = F64(s + 8), c = F64(s + len - 8) * mul, d = F64(s + len - 16) * K2;
  return hl16(rot(a + b, 43) + rot(c, 30) + d, a + rot(b + K2, 18) + c, mul);
}

static uint64_t h33to64(const uint8_t* s, uint64_t len) {
  uint64_t mul = K2 + len * 2;
  uint64_t a = F64(s) * K2, b = F64(s + 8), c = F64(s + len - 8) * mul, d = F64(s + len - 16) * K2;
  uint64_t y = rot(a + b, 43) + rot(c, 30) + d;
  uint64_t z = hl16(y, a + rot(b + K2, 18) + c, mul);
  uint64_t e = F64(s + 16) * mul, f = F64(s + 24);
  uint64_t g = (y + F64(s + len - 32)) * mul, h = (z + F64(s + len - 24)) * mul;
  return hl16(rot(e + f, 43) + rot(g, 30) + h, e + rot(f + a, 18) + g, mul);
}

/* WeakHashLen32WithSeeds(s[0..31], a, b) -> (*first, *second) */
static void weak32(const uint8_t* s, uint64_t a, uint64_t b, uint64_t* first, uint64_t* second) {
  uint64_t w = F64(s), x = F64(s + 8), y = F64(s + 16), z = F64(s + 24);
  a += w;
  b = rot(b + a + z, 21);
  uint64_t c = a;
  a += x;
  a += y;
  b += rot(a, 44);
  *first = a + z;
  *second = b + c;
}

uint64_t ho_fingerprint64(const uint8_t* s, int64_t n) {
  const uint64_t len = (uint64_t)n, seed = 81;
  if (len <= 16) return h0to16(s, len);
  if (len <= 32) return h17to32(s, len);
  if (len <= 64) return h33to64(s, len);
  uint64_t x = seed, y = seed * K1 + 113, z = smix(y * K2 + 113) * K2, t;
  uint64_t v1 = 0, v2 = 0, w1 = 0, w2 = 0;
  x = x * K2 + F64(s);
  const uint8_t* end = s + ((len - 1) / 64) * 64;
  const uint8_t* last64 = end + ((len - 1) & 63) - 63;
  do {
    x = rot(x + y + v1 + F64(s + 8), 37) * K1;
    y = rot(y + v2 + F64(s + 48), 42) * K1;
    x ^= w2;
    y += v1 + F64(s + 40);
    z = rot(z + w1, 33) * K1;
    weak32(s, v2 * K1, x + w1, &v1, &v2);
    weak32(s + 32, z + w2, y + F64(s + 16), &w1, &w2);
    t = z; z = x; x = t;
    s += 64;
  } while (s != end);
  uint64_t mul = K1 + ((z & 0xff) << 1);
  s = last64;
  w1 += ((len - 1) & 63);
  v1 += w1;
  w1 += v1;
  x = rot(x + y + v1 + F64(s + 8), 37) * mul;
  y = rot(y + v2 + F64(s + 48), 42) * mul;
  x ^= w2 * 9;
  y += v1 * 9 + F64(s + 40);
  z = rot(z + w1, 33) * mul;
  weak32(s, v2 * mul, x + w1, &v1, &v2);
  weak32(s + 32, z + w2, y + F64(s + 16), &w1, &w2);
  t = z; z = x; x = t;
  return hl16(hl16(v1, w1, mul) + smix(y) * K0 + z, hl16(v2, w2, mul) + x, mul);
}

static uint64_t hash_msg(const uint8_t* m, int64_t len, int salted, uint64_t k0, uint64_t k1) {
  return salted ? uo_siphash(k0, k1, m, len) : ho_fingerprint64(m, len);
}

static int64_t to_bin(uint64_t h, int is_mask, uint64_t num_bins, int has_mask) {
  if (has_mask && num_bins > 1) return is_mask ? 0 : (int64_t)(1 + h % (num_bins - 1));
  return (int64_t)(h % num_bins);
}

void ho_hash_i64(const int64_t* v, int64_t n, int salted, uint64_t k0, uint64_t k1, uint64_t num_bins, int has_mask,
                 int64_t mask, int64_t* out) {
  char buf[24];
  for (int64_t i = 0; i < n; ++i) {
    int len = uo_as_string(v[i], buf);
    out[i] = to_bin(hash_msg((const uint8_t*)buf, len, salted, k0, k1), v[i] == mask, num_bins, has_mask);
  }
}

void ho_hash_bytes(const uint8_t* bytes, const int64_t* off, int64_t n, int salted, uint64_t k0, uint64_t k1,
                   uint64_t num_bins, int has_mask, const uint8_t* mask, int64_t mask_len, int64_t* out) {
  for (int64_t i = 0; i < n; ++i) {
    const uint8_t* s = bytes + off[i];
    int64_t len = off[i + 1] - off[i];
    int is_mask = len == mask_len && (len == 0 || memcmp(s, mask, (size_t)len) == 0);
    out[i] = to_bin(hash_msg(s, len, salted, k0, k1), is_mask, num_bins, has_mask);
  }
}
