// bdiff_philox.cuh — counter-based Gaussian noise: Philox4x32-10 (Salmon et al., SC'11) and Box-Muller.  Every value is
// a pure function of (seed, draw, element); the layout is the one include/bdiff.h documents for bdiff_noise_fill.
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

namespace bdiff {

struct Philox4 {
  uint32_t w[4];
};

__device__ __forceinline__ Philox4 philox4x32_10(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3, uint32_t k0,
                                                 uint32_t k1) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const uint32_t hi0 = __umulhi(0xD2511F53u, c0), lo0 = 0xD2511F53u * c0;
    const uint32_t hi1 = __umulhi(0xCD9E8D57u, c2), lo1 = 0xCD9E8D57u * c2;
    const uint32_t n0 = hi1 ^ c1 ^ k0, n2 = hi0 ^ c3 ^ k1;
    c0 = n0; c1 = lo1; c2 = n2; c3 = lo0;
    k0 += 0x9E3779B9u;
    k1 += 0xBB67AE85u;
  }
  return Philox4{{c0, c1, c2, c3}};
}

// Block `block` of draw `draw`: counter {block lo, block hi, draw lo, draw hi}, key {seed lo, seed hi}.
__device__ __forceinline__ Philox4 philox_block(uint64_t seed, uint64_t draw, uint64_t block) {
  return philox4x32_10((uint32_t)block, (uint32_t)(block >> 32), (uint32_t)draw, (uint32_t)(draw >> 32), (uint32_t)seed,
                       (uint32_t)(seed >> 32));
}

// Element e of draw `draw`: Box-Muller on the word pair (e & 2, e | 1) of block e >> 2, cosine for even e, sine for odd.
__device__ __forceinline__ float philox_normal(uint64_t seed, uint64_t draw, uint64_t e) {
  const Philox4 b = philox_block(seed, draw, e >> 2);
  const int j = (int)(e & 3);
  const uint32_t wu = b.w[j & 2], wv = b.w[j | 1];
  const double u = ((double)wu + 0.5) * 0x1p-32;               // (0, 1): log stays finite
  const double r = sqrt(__dmul_rn(-2.0, log(u)));
  double sn, cs;
  sincospi((double)wv * 0x1p-31, &sn, &cs);                   // angle 2 pi wv 2^-32
  return (float)__dmul_rn(r, (j & 1) ? sn : cs);
}

}  // namespace bdiff
