// Gaussian noise for client-level differential privacy (DP-FedAvg): Philox4x32-10 and Box-Muller as device functions.
//
// z[i] is a pure function of (seed, round, i): Philox4x32-10 with key (seed_lo, seed_hi) and counter
// (q_lo, q_hi, round, 0), q = i / 4, gives four 32-bit words x0..x3; u = (x + 0.5) * 2^-32 maps them into (0, 1), and
// Box-Muller on (x0, x1) and (x2, x3) gives z[4q .. 4q+3].  The constants and round structure are those of cuRAND's
// curand_Philox4x32_10 (Salmon et al., SC'11), so the stream can be reproduced on the host (baton_b200/parallel/dp.py)
// and does not depend on how the elements are split over threads, CTAs, tiles or ranks.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace b200 {

__device__ __forceinline__ uint4 philox4x32_10(uint4 c, uint2 k) {
  constexpr uint32_t M0 = 0xD2511F53u, M1 = 0xCD9E8D57u, W0 = 0x9E3779B9u, W1 = 0xBB67AE85u;
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const uint32_t lo0 = M0 * c.x, hi0 = __umulhi(M0, c.x);
    const uint32_t lo1 = M1 * c.z, hi1 = __umulhi(M1, c.z);
    c = make_uint4(hi1 ^ c.y ^ k.x, lo1, hi0 ^ c.w ^ k.y, lo0);
    k.x += W0;
    k.y += W1;
  }
  return c;
}

// Box-Muller on one pair of words.  The logarithm is taken in double: the build's --use_fast_math turns logf into an
// approximation whose absolute error near u = 1 would dominate the small radii.  The angle uses sincospif (exact
// argument reduction); the result still differs from the host reference in the last bits, so tests compare to a tolerance.
__device__ __forceinline__ float2 box_muller(uint32_t a, uint32_t b) {
  const double u1 = (static_cast<double>(a) + 0.5) * 2.3283064365386963e-10;    // 2^-32
  const float u2 = (static_cast<float>(b) + 0.5f) * 2.3283064365386963e-10f;
  const float r = static_cast<float>(sqrt(-2.0 * log(u1)));
  float s, c;
  sincospif(2.f * u2, &s, &c);
  return make_float2(r * c, r * s);
}

// z[4q .. 4q+3] of the stream (seed, round)
__device__ __forceinline__ float4 dp_normal4(unsigned long long seed, uint32_t round, unsigned long long q) {
  const uint4 x = philox4x32_10(make_uint4(static_cast<uint32_t>(q), static_cast<uint32_t>(q >> 32), round, 0u),
                                make_uint2(static_cast<uint32_t>(seed), static_cast<uint32_t>(seed >> 32)));
  const float2 z01 = box_muller(x.x, x.y), z23 = box_muller(x.z, x.w);
  return make_float4(z01.x, z01.y, z23.x, z23.y);
}

}  // namespace b200
