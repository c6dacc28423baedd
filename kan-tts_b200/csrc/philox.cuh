// Philox4x32-10 (Salmon et al., "Parallel random numbers: as easy as 1, 2, 3", SC 2011): a counter-based generator,
// one 128-bit block of random bits per (counter, key), no state.  The constants and round structure are Random123's;
// oracle/nsf.py restates it in NumPy and checks the Random123 known-answer vectors.
#pragma once
#include <stdint.h>

namespace kt {

struct Philox4 {
  uint32_t v[4];
};

__host__ __device__ __forceinline__ Philox4 philox4x32_10(Philox4 c, uint32_t k0, uint32_t k1) {
  constexpr uint32_t kM0 = 0xD2511F53u, kM1 = 0xCD9E8D57u, kW0 = 0x9E3779B9u, kW1 = 0xBB67AE85u;
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    if (r > 0) { k0 += kW0; k1 += kW1; }
    const uint64_t p0 = (uint64_t)kM0 * c.v[0], p1 = (uint64_t)kM1 * c.v[2];
    const uint32_t hi0 = (uint32_t)(p0 >> 32), lo0 = (uint32_t)p0, hi1 = (uint32_t)(p1 >> 32), lo1 = (uint32_t)p1;
    c = Philox4{{hi1 ^ c.v[1] ^ k0, lo1, hi0 ^ c.v[3] ^ k1, lo0}};
  }
  return c;
}

}  // namespace kt
