// The in-kernel normal generator shared by TD3's target smoothing (td3.cu) and the actors' exploration noise
// (policy.cu): Philox4x32-10 words, mapped to (0, 1) and through Box-Muller.  Each caller keys its own stream; see
// include/r2d2_b200.h (r2d2_target_smoothing, r2d2_exploration).
#pragma once
#include <stdint.h>

namespace r2d2 {

// Philox4x32-10 (Salmon et al., "Parallel random numbers: as easy as 1, 2, 3", SC'11): ten rounds, the key bumped
// between rounds.  Known-answer vectors are checked in tests/test_cpu_td3.py (oracle) and tests/test_gpu_td3.py.
struct Philox4 { uint32_t x[4]; };

__device__ __forceinline__ Philox4 philox4x32_10(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3, uint32_t k0,
                                                 uint32_t k1) {
  constexpr uint32_t M0 = 0xD2511F53u, M1 = 0xCD9E8D57u, W0 = 0x9E3779B9u, W1 = 0xBB67AE85u;
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    if (r) { k0 += W0; k1 += W1; }
    const uint32_t hi0 = __umulhi(M0, c0), lo0 = M0 * c0;
    const uint32_t hi1 = __umulhi(M1, c2), lo1 = M1 * c2;
    const uint32_t n0 = hi1 ^ c1 ^ k0, n2 = hi0 ^ c3 ^ k1;
    c0 = n0; c1 = lo1; c2 = n2; c3 = lo0;
  }
  return Philox4{{c0, c1, c2, c3}};
}

// (0, 1), exact: the top 23 bits as an odd multiple of 2^-24
__device__ __forceinline__ float unit_open(uint32_t x) { return (float)(2u * (x >> 9) + 1u) * 0x1p-24f; }

// Box-Muller on one pair of words (xa, xb): the pair's two normals are rad * c (even element) and rad * s (odd), with
// rad = sqrt(-2 ln u_a) and (s, c) = sincos(2 pi u_b), in fp32 with precise logf, sqrtf and sincospif
__device__ __forceinline__ void box_muller(uint32_t xa, uint32_t xb, float& rad, float& s, float& c) {
  const float u1 = unit_open(xa), u2 = unit_open(xb);
  rad = sqrtf(-2.0f * logf(u1));
  sincospif(2.0f * u2, &s, &c);
}

}  // namespace r2d2
