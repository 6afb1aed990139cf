// siphash.cuh -- SipHash-2-4 on the device, shared by K8 (unified_embedding.cu: tf-keras Hashing's bucket of a value) and
// K15 (lookup.cu: the slot and fingerprint of a vocabulary string).
//
// A message up to SIP_SHORT bytes is formed once into a 192-bit little-endian register (three uint64) and hashed from
// there; a longer one is hashed from memory (`p`, `len` bytes).
#pragma once
#include <stdint.h>

namespace tfrs {

constexpr int SIP_SHORT = 23;           // messages up to this many bytes live in three 64-bit registers

__device__ __forceinline__ uint64_t rotl(uint64_t x, int b) { return (x << b) | (x >> (64 - b)); }

struct Sip {
  uint64_t v0, v1, v2, v3;
  __device__ __forceinline__ Sip(uint64_t k0, uint64_t k1)
      : v0(k0 ^ 0x736f6d6570736575ull), v1(k1 ^ 0x646f72616e646f6dull), v2(k0 ^ 0x6c7967656e657261ull),
        v3(k1 ^ 0x7465646279746573ull) {}
  __device__ __forceinline__ void round() {
    v0 += v1; v1 = rotl(v1, 13); v1 ^= v0; v0 = rotl(v0, 32);
    v2 += v3; v3 = rotl(v3, 16); v3 ^= v2;
    v0 += v3; v3 = rotl(v3, 21); v3 ^= v0;
    v2 += v1; v1 = rotl(v1, 17); v1 ^= v2; v2 = rotl(v2, 32);
  }
  __device__ __forceinline__ void block(uint64_t m) { v3 ^= m; round(); round(); v0 ^= m; }
  __device__ __forceinline__ uint64_t finish() { v2 ^= 0xff; round(); round(); round(); round(); return v0 ^ v1 ^ v2 ^ v3; }
};

// 192-bit little-endian message register: push(c) shifts every byte up by one and puts c at byte 0
struct Msg {
  uint64_t w0 = 0, w1 = 0, w2 = 0;
  int len = 0;
  __device__ __forceinline__ void push(uint32_t c) {
    w2 = (w2 << 8) | (w1 >> 56); w1 = (w1 << 8) | (w0 >> 56); w0 = (w0 << 8) | c; ++len;
  }
};

__device__ __forceinline__ uint64_t load_word(const uint8_t* p, int nbytes) {
  uint64_t w = 0;
  for (int k = nbytes - 1; k >= 0; --k) w = (w << 8) | p[k];
  return w;
}

// SipHash-2-4 of a formed message: short ones from registers, longer strings from memory (`p`, `len` bytes).
__device__ __forceinline__ uint64_t siphash(const Msg& m, const uint8_t* p, uint64_t k0, uint64_t k1) {
  Sip s(k0, k1);
  const int nb = m.len >> 3;
  uint64_t last;
  if (m.len <= SIP_SHORT) {
    if (nb > 0) s.block(m.w0);
    if (nb > 1) s.block(m.w1);
    last = nb == 0 ? m.w0 : (nb == 1 ? m.w1 : m.w2);
  } else {
    for (int b = 0; b < nb; ++b) s.block(load_word(p + 8 * b, 8));
    last = load_word(p + 8 * nb, m.len & 7);
  }
  s.block(last | ((uint64_t)(m.len & 0xff) << 56));
  return s.finish();
}

// Forms into the empty message m the byte string b[0, len): up to SIP_SHORT bytes loaded into the register, a longer one
// left in memory (*p = b; *p stays untouched for a short one).
__device__ __forceinline__ void bytes_msg(Msg& m, const uint8_t* b, long long len, const uint8_t** p) {
  if (len <= SIP_SHORT) {
    for (int k = (int)len - 1; k >= 0; --k) m.push(b[k]);
  } else {
    m.len = (int)min(len, (long long)INT32_MAX);
    *p = b;
  }
}

}  // namespace tfrs
