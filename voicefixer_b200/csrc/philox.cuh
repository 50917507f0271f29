// Philox4x32-10 (Salmon, Moraes, Dror, Shaw, "Parallel random numbers: as easy as 1, 2, 3", SC'11): the counter-based
// generator of curand_Philox4x32_10, as a pure function of (counter, key).  Mode 2's seeded dropout draws its keep bits
// from it (dropout_seeded_kernel, DESIGN.md §3); voicefixer_b200/philox.py restates it on the host.
#pragma once
#include <stdint.h>

namespace vfx {

struct philox4 { uint32_t w[4]; };

__device__ __forceinline__ void philox_round(uint32_t (&c)[4], uint32_t k0, uint32_t k1) {
  const uint32_t hi0 = __umulhi(0xD2511F53u, c[0]), lo0 = 0xD2511F53u * c[0];
  const uint32_t hi1 = __umulhi(0xCD9E8D57u, c[2]), lo1 = 0xCD9E8D57u * c[2];
  const uint32_t n0 = hi1 ^ c[1] ^ k0, n2 = hi0 ^ c[3] ^ k1;
  c[0] = n0; c[1] = lo1; c[2] = n2; c[3] = lo0;
}

// Ten rounds, the key bumped by the Weyl constants between them.  Straight-line code: the caller keeps it out of loops
// whose trip count ptxas does not know, so that the four words and two key halves stay in registers.
__device__ __forceinline__ philox4 philox4x32_10(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3, uint32_t k0,
                                                 uint32_t k1) {
  uint32_t c[4] = {c0, c1, c2, c3};
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    philox_round(c, k0, k1);
    k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
  }
  return philox4{{c[0], c[1], c[2], c[3]}};
}

}  // namespace vfx
