// wdb_noisy.cuh -- the one definition of a noisy network's noise element (include/wdb200.h,
// wdb_noisy_*): every kernel that draws noisy-head noise calls noisy_f.
#pragma once
#include "wdb_common.cuh"

namespace wdb {

constexpr uint32_t kNoisyTag = 0x4E000000u;   // keeps the counters apart from every other draw

// f(eps) = sgn(eps) sqrt(|eps|) of noise element e of noisy layer `layer`, counter row `row`,
// in (domain, count): eps = u32x2_to_normal of Philox4x32-10 words (x, y) for even e and (z, w)
// for odd e.
__device__ __forceinline__ float noisy_f(unsigned long long seed, int domain,
                                         unsigned long long count, uint32_t row, int layer,
                                         int e) {
  const uint4 c = make_uint4((uint32_t)count,
                             kNoisyTag | ((uint32_t)domain << 16) |
                                 ((uint32_t)(count >> 32) & 0xFFFFu),
                             row, ((uint32_t)layer << 16) | ((uint32_t)e >> 1));
  const uint4 w = philox4x32_10(c, make_uint2((uint32_t)seed, (uint32_t)(seed >> 32)));
  const float n = (e & 1) ? u32x2_to_normal(w.z, w.w) : u32x2_to_normal(w.x, w.y);
  return copysignf(sqrtf(fabsf(n)), n);
}

}  // namespace wdb
