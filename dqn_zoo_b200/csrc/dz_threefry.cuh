// Threefry-2x32, 20 rounds (Salmon et al., "Parallel random numbers: as easy as 1, 2, 3"): the counter-based generator
// behind jax.random at the pinned jax 0.3.10 (dz_jaxprng.cu) and the randomness of the device games (dz_game.cuh).
// One definition, compiled for the host and the device; its known answers are in dz_jaxprng.cu.
#pragma once
#include <stdint.h>

namespace dz {

__host__ __device__ __forceinline__ uint32_t rotl32(uint32_t x, int r) { return (x << r) | (x >> (32 - r)); }

__host__ __device__ inline void threefry2x32(uint32_t k0, uint32_t k1, uint32_t c0, uint32_t c1, uint32_t* o0, uint32_t* o1) {
  const uint32_t ks[3] = {k0, k1, k0 ^ k1 ^ 0x1BD11BDAu};
  const int rot[2][4] = {{13, 15, 26, 6}, {17, 29, 16, 24}};
  uint32_t x0 = c0 + ks[0], x1 = c1 + ks[1];
#pragma unroll
  for (int i = 0; i < 5; ++i) {
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      x0 += x1;
      x1 = rotl32(x1, rot[i & 1][j]);
      x1 ^= x0;
    }
    x0 += ks[(i + 1) % 3];
    x1 += ks[(i + 2) % 3] + (uint32_t)(i + 1);
  }
  *o0 = x0;
  *o1 = x1;
}

}  // namespace dz
