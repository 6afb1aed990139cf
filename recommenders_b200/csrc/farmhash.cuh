// farmhash.cuh -- FarmHash Fingerprint64 (farmhashna::Hash64 of the published FarmHash) on the device: the hash of
// tf.strings.to_hash_bucket_fast, which buckets an unsalted tf-keras Hashing (K18, hashing.cu).
//
// The 1-3, 4-7 and 8-16 byte branches are pinned by TF's published examples; the 17-32, 33-64 and > 64 byte branches are
// restated from the published algorithm and unpinned against TF (DESIGN.md §2, A22).
//
// The hash reads its message only through a source S: S::u8(k) is byte k, S::f32(k) / S::f64(k) are the little-endian 4 /
// 8 bytes at byte offset k.  Strings start at any byte offset, so no source dereferences a pointer wider than a byte made
// from one: ByteSrc builds every fetch from byte loads, MsgSrc shifts the words of a message register (bucket.cuh).
#pragma once
#include <stdint.h>

namespace tfrs {
namespace farm {

constexpr uint64_t k0 = 0xc3a5c85c97cb3127ull, k1 = 0xb492b66fbe98f273ull, k2 = 0x9ae16a3b2f90404full;

// Bytes in device memory at any alignment.
struct ByteSrc {
  const uint8_t* b;
  __device__ __forceinline__ uint32_t u8(long long k) const { return __ldg(b + k); }
  __device__ __forceinline__ uint64_t f32(long long k) const {
    return u8(k) | (u8(k + 1) << 8) | (u8(k + 2) << 16) | ((uint64_t)u8(k + 3) << 24);
  }
  __device__ __forceinline__ uint64_t f64(long long k) const { return f32(k) | (f32(k + 4) << 32); }
};

// A message of at most 24 bytes held little-endian in three registers (a Msg).  Bytes past its length are zero.
struct MsgSrc {
  uint64_t w0, w1, w2;
  __device__ __forceinline__ uint64_t word(long long j) const { return j == 0 ? w0 : (j == 1 ? w1 : (j == 2 ? w2 : 0)); }
  __device__ __forceinline__ uint64_t f64(long long k) const {
    const int sh = (int)(k & 7) * 8;
    const uint64_t lo = word(k >> 3);
    return sh ? (lo >> sh) | (word((k >> 3) + 1) << (64 - sh)) : lo;
  }
  __device__ __forceinline__ uint64_t f32(long long k) const { return f64(k) & 0xffffffffull; }
  __device__ __forceinline__ uint32_t u8(long long k) const { return (uint32_t)(word(k >> 3) >> ((k & 7) * 8)) & 0xffu; }
};

__device__ __forceinline__ uint64_t rot(uint64_t v, int s) { return (v >> s) | (v << (64 - s)); }   // 0 < s < 64
__device__ __forceinline__ uint64_t shift_mix(uint64_t v) { return v ^ (v >> 47); }

__device__ __forceinline__ uint64_t len16(uint64_t u, uint64_t v, uint64_t mul) {
  uint64_t a = (u ^ v) * mul;
  a ^= a >> 47;
  uint64_t b = (v ^ a) * mul;
  b ^= b >> 47;
  return b * mul;
}

template <class S>
__device__ __forceinline__ uint64_t len0to16(const S& s, uint64_t len) {
  if (len >= 8) {
    const uint64_t mul = k2 + len * 2;
    const uint64_t a = s.f64(0) + k2;
    const uint64_t b = s.f64(len - 8);
    const uint64_t c = rot(b, 37) * mul + a;
    const uint64_t d = (rot(a, 25) + b) * mul;
    return len16(c, d, mul);
  }
  if (len >= 4) {
    const uint64_t mul = k2 + len * 2;
    return len16(len + (s.f32(0) << 3), s.f32(len - 4), mul);
  }
  if (len > 0) {
    const uint32_t y = s.u8(0) + (s.u8(len >> 1) << 8);
    const uint32_t z = (uint32_t)len + (s.u8(len - 1) << 2);
    return shift_mix(y * k2 ^ z * k0) * k2;
  }
  return k2;
}

template <class S>
__device__ __forceinline__ uint64_t len17to32(const S& s, uint64_t len) {
  const uint64_t mul = k2 + len * 2;
  const uint64_t a = s.f64(0) * k1;
  const uint64_t b = s.f64(8);
  const uint64_t c = s.f64(len - 8) * mul;
  const uint64_t d = s.f64(len - 16) * k2;
  return len16(rot(a + b, 43) + rot(c, 30) + d, a + rot(b + k2, 18) + c, mul);
}

template <class S>
__device__ __forceinline__ uint64_t len33to64(const S& s, uint64_t len) {
  const uint64_t mul = k2 + len * 2;
  const uint64_t a = s.f64(0) * k2;
  const uint64_t b = s.f64(8);
  const uint64_t c = s.f64(len - 8) * mul;
  const uint64_t d = s.f64(len - 16) * k2;
  const uint64_t y = rot(a + b, 43) + rot(c, 30) + d;
  const uint64_t z = len16(y, a + rot(b + k2, 18) + c, mul);
  const uint64_t e = s.f64(16) * mul;
  const uint64_t f = s.f64(24);
  const uint64_t g = (y + s.f64(len - 32)) * mul;
  const uint64_t h = (z + s.f64(len - 24)) * mul;
  return len16(rot(e + f, 43) + rot(g, 30) + h, e + rot(f + a, 18) + g, mul);
}

// WeakHashLen32WithSeeds of the 32 bytes at offset p, seeds a and b: (first, second) returned in *x, *y.
template <class S>
__device__ __forceinline__ void weak32(const S& s, long long p, uint64_t a, uint64_t b, uint64_t* x, uint64_t* y) {
  const uint64_t w = s.f64(p), v1 = s.f64(p + 8), v2 = s.f64(p + 16), z = s.f64(p + 24);
  a += w;
  b = rot(b + a + z, 21);
  const uint64_t c = a;
  a += v1;
  a += v2;
  b += rot(a, 44);
  *x = a + z;
  *y = b + c;
}

// len > 64: 64-byte blocks from the start, then the last 64 bytes.
template <class S>
__device__ __forceinline__ uint64_t len65plus(const S& s, uint64_t len) {
  const uint64_t seed = 81;
  uint64_t x = seed, y = seed * k1 + 113, z = shift_mix(y * k2 + 113) * k2;
  uint64_t v0 = 0, v1 = 0, w0 = 0, w1 = 0;
  x = x * k2 + s.f64(0);
  const long long end = (long long)((len - 1) / 64) * 64;
  for (long long p = 0; p != end; p += 64) {
    x = rot(x + y + v0 + s.f64(p + 8), 37) * k1;
    y = rot(y + v1 + s.f64(p + 48), 42) * k1;
    x ^= w1;
    y += v0 + s.f64(p + 40);
    z = rot(z + w0, 33) * k1;
    weak32(s, p, v1 * k1, x + w0, &v0, &v1);
    weak32(s, p + 32, z + w1, y + s.f64(p + 16), &w0, &w1);
    const uint64_t t = z; z = x; x = t;
  }
  const uint64_t mul = k1 + ((z & 0xff) << 1);
  const long long p = (long long)len - 64;
  w0 += (len - 1) & 63;
  v0 += w0;
  w0 += v0;
  x = rot(x + y + v0 + s.f64(p + 8), 37) * mul;
  y = rot(y + v1 + s.f64(p + 48), 42) * mul;
  x ^= w1 * 9;
  y += v0 * 9 + s.f64(p + 40);
  z = rot(z + w0, 33) * mul;
  weak32(s, p, v1 * mul, x + w0, &v0, &v1);
  weak32(s, p + 32, z + w1, y + s.f64(p + 16), &w0, &w1);
  const uint64_t t = z; z = x; x = t;
  return len16(len16(v0, w0, mul) + shift_mix(y) * k0 + z, len16(v1, w1, mul) + x, mul);
}

}  // namespace farm

// Fingerprint64 of a message of at most 32 bytes (the decimal text of an int64 is at most 20).
template <class S>
__device__ __forceinline__ uint64_t fingerprint64_short(const S& s, uint64_t len) {
  return len <= 16 ? farm::len0to16(s, len) : farm::len17to32(s, len);
}

template <class S>
__device__ __forceinline__ uint64_t fingerprint64(const S& s, uint64_t len) {
  if (len <= 32) return fingerprint64_short(s, len);
  return len <= 64 ? farm::len33to64(s, len) : farm::len65plus(s, len);
}

}  // namespace tfrs
