// bucket.cuh -- the message and the bin arithmetic of tf-keras Hashing, shared by K8 (unified_embedding.cu, salted
// buckets fused with the row gather) and K18 (hashing.cu, the Hashing layer's bins).
#pragma once
#include <stdint.h>
#include "siphash.cuh"

namespace tfrs {

// x mod d with magic = floor((2^64 - 1) / d), d >= 1: the estimate q = hi64(x * magic) is at most 2 below floor(x / d)
// (DESIGN.md K8), so two conditional subtractions make the remainder exact for every d < 2^64.
__device__ __forceinline__ uint64_t mod_magic(uint64_t x, uint64_t d, uint64_t magic) {
  uint64_t r = x - __umul64hi(x, magic) * d;
  if (r >= d) r -= d;
  if (r >= d) r -= d;
  return r;
}

// tf.as_string of an int64: digits generated least significant first and pushed at byte 0, so the most significant
// digit ends at byte 0.  |x| is split into 32-bit pieces below 10^9.
__device__ __forceinline__ Msg decimal_msg(long long x) {
  Msg m;
  const bool neg = x < 0;
  const uint64_t u = neg ? 0ull - (uint64_t)x : (uint64_t)x;
  const uint64_t q1 = u / 1000000000ull;
  const uint64_t q2 = q1 / 1000000000ull;
  const uint32_t piece[3] = {(uint32_t)(u - q1 * 1000000000ull), (uint32_t)(q1 - q2 * 1000000000ull), (uint32_t)q2};
  const int top = q2 ? 2 : (q1 ? 1 : 0);
#pragma unroll
  for (int p = 0; p < 3; ++p) {
    if (p > top) break;
    uint32_t v = piece[p];
#pragma unroll
    for (int k = 0; k < 9; ++k) {
      if (p == top && k > 0 && v == 0) break;    // the leading piece has no leading zeros
      const uint32_t q = v / 10u;
      m.push('0' + (v - q * 10u));
      v = q;
    }
  }
  if (neg) m.push('-');
  return m;
}

}  // namespace tfrs
