// philox.cuh -- Philox4x32-10 (Salmon et al., "Parallel random numbers: as easy as 1, 2, 3", SC'11) with the standard
// multipliers M = (0xD2511F53, 0xCD9E8D57) and Weyl key increments W = (0x9E3779B9, 0xBB67AE85): ten rounds, the key
// bumped by W before every round but the first.  Counter-based: the output is a pure function of (counter, key), so a
// backward pass regenerates a forward's random words instead of storing them.
#pragma once
#include <stdint.h>

namespace tfrs {

__device__ __forceinline__ uint4 philox4x32_10(uint4 c, uint32_t k0, uint32_t k1) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    if (r > 0) {
      k0 += 0x9E3779B9u;
      k1 += 0xBB67AE85u;
    }
    const uint32_t lo0 = 0xD2511F53u * c.x, hi0 = __umulhi(0xD2511F53u, c.x);
    const uint32_t lo1 = 0xCD9E8D57u * c.z, hi1 = __umulhi(0xCD9E8D57u, c.z);
    c = make_uint4(hi1 ^ c.y ^ k0, lo1, hi0 ^ c.w ^ k1, lo0);
  }
  return c;
}

}  // namespace tfrs
