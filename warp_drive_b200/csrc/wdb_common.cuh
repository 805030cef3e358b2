// wdb_common.cuh -- shared device helpers for libwdb200.so (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/wdb200.h"

#if defined(__CUDA_ARCH__) && (__CUDA_ARCH__ != 900)
#error "libwdb200 targets sm_90a (H100) only"
#endif

#define WDB_API extern "C" __attribute__((visibility("default")))

namespace wdb {

extern long long g_launch_count;

inline int finish_launch() {
  ++g_launch_count;
  return static_cast<int>(cudaGetLastError());
}

inline cudaStream_t as_stream(void *s) { return reinterpret_cast<cudaStream_t>(s); }

constexpr int kWarp = 32;
constexpr int kNumSMs = 132;  // H100 SXM

inline int round_up(int v, int m) { return (v + m - 1) / m * m; }

// ----------------------------------------------------------------------------
// Philox4x32-10 (Salmon et al. SC'11).  Counter-based: no per-thread state besides
// a 64-bit draw offset, so the whole RNG "state" is one coalesced u64 per stream.
// Pinned bit-for-bit by the Random123 known-answer vectors (tests/test_rng.py).
// ----------------------------------------------------------------------------
struct RngHeader {
  unsigned long long seed;
  unsigned long long n_streams;
};

__device__ __forceinline__ uint4 philox4x32_10(uint4 c, uint2 k) {
#pragma unroll
  for (int r = 0; r < 10; r++) {
    const uint32_t hi0 = __umulhi(0xD2511F53u, c.x);
    const uint32_t lo0 = 0xD2511F53u * c.x;
    const uint32_t hi1 = __umulhi(0xCD9E8D57u, c.z);
    const uint32_t lo1 = 0xCD9E8D57u * c.z;
    c = make_uint4(hi1 ^ c.y ^ k.x, lo1, hi0 ^ c.w ^ k.y, lo0);
    k.x += 0x9E3779B9u;
    k.y += 0xBB67AE85u;
  }
  return c;
}

// Four 32-bit draws for (stream, offset); the caller bumps the offset.
__device__ __forceinline__ uint4 rng_draw4(const RngHeader &h, unsigned long long stream,
                                           unsigned long long offset) {
  const uint4 ctr = make_uint4((uint32_t)offset, (uint32_t)(offset >> 32),
                               (uint32_t)stream, (uint32_t)(stream >> 32));
  const uint2 key = make_uint2((uint32_t)h.seed, (uint32_t)(h.seed >> 32));
  return philox4x32_10(ctr, key);
}

// u32 -> (0, 1], the same mapping as curand_uniform (x * 2^-32 + 2^-33), which is what
// the reference sampler draws (random.cu:72).
__device__ __forceinline__ float u32_to_uniform(uint32_t x) {
  return x * 2.3283064365386963e-10f + 1.1641532182693481e-10f;
}

// Box-Muller on two (0,1] uniforms -> one N(0,1) draw.
__device__ __forceinline__ float u32x2_to_normal(uint32_t a, uint32_t b) {
  const float u1 = u32_to_uniform(a);
  const float u2 = u32_to_uniform(b);
  return sqrtf(-2.0f * logf(u1)) * cosf(6.2831853071795864f * u2);
}

// Source row of reset descriptor `d` for `env`: the env's own row, or from a reset pool
// (pool_rows > 0) a draw p of the env's pool stream at pool_off + n_pool and row =
// int(p * pool_rows) (pool_reset.py:24-27), clamped for the p == 1.0 edge of (0, 1].
// n_pool counts the pool draws of this reset; it advances for pool descriptors only.
__device__ __forceinline__ long long reset_src_row(const wdb_reset_desc &d, const RngHeader &h,
                                                   int env, unsigned long long pool_off,
                                                   int &n_pool) {
  if (d.pool_rows <= 0) return env;
  const float p = u32_to_uniform(rng_draw4(h, (unsigned long long)env, pool_off + n_pool).x);
  const long long row = (long long)(p * (float)d.pool_rows);
  n_pool++;
  return row < d.pool_rows ? row : d.pool_rows - 1;
}

__device__ __forceinline__ unsigned long long *rng_offsets(void *rng_state) {
  return reinterpret_cast<unsigned long long *>(
      reinterpret_cast<char *>(rng_state) + sizeof(RngHeader));
}

// ----------------------------------------------------------------------------
// Categorical index selection, bit-faithful to the reference's search_index
// (warp_drive/cuda_includes/core/random.cu:33-49) over a float32 CDF.
// ----------------------------------------------------------------------------
__device__ __forceinline__ int search_index(const float *cdf, int stride, float p, int r) {
  int left = 0, right = r;
  while (left <= right) {
    const int mid = left + (right - left) / 2;
    const float v = cdf[mid * stride];
    if (fabsf(v - p) < 1.0e-8f) return mid;
    if (v < p) left = mid + 1; else right = mid - 1;
  }
  return left > r ? r : left;
}

// Categorical draw from one probability row held in registers, p[0 .. A) with A <= kMax <=
// 32: the float32 CDF of the same left-to-right additions (never contracted into an FMA with
// whatever produced p) searched exactly as search_index(cdf, 1, u, A - 1) searches it.  That
// search only asks two things of an entry it probes, |cdf - u| < 1e-8 and cdf < u, so both
// are evaluated for every entry as bit masks first and the search then runs on the masks:
// no dynamically indexed register array.  The packed TagContinuous step and the policy
// forward (wdb_mlp_policy_forward_sampled) both sample through this, so they draw the same
// action from the same probabilities and uniform.
template <int kMax>
__device__ __forceinline__ int sample_cdf_regs(const float (&p)[kMax], int A, float u) {
  static_assert(kMax <= 32, "one bit per action");
  uint32_t near = 0, below = 0;
  float c = 0.0f;
#pragma unroll
  for (int i = 0; i < kMax; i++) {
    c = i ? __fadd_rn(p[i], c) : p[i];
    if (i < A) {
      near |= (fabsf(__fsub_rn(c, u)) < 1.0e-8f ? 1u : 0u) << i;
      below |= (c < u ? 1u : 0u) << i;
    }
  }
  const int r = A - 1;
  int left = 0, right = r;
  while (left <= right) {
    const int mid = left + (right - left) / 2;
    if ((near >> mid) & 1u) return mid;
    if ((below >> mid) & 1u) left = mid + 1; else right = mid - 1;
  }
  return left > r ? r : left;
}

// Index selection for masked policies: p[0 .. A) becomes the same float32 CDF the reference
// sampler builds, and the result is the first index with p_i > 0 whose CDF reaches u, or,
// when u lies above the float32 total, the last index with p_i > 0.  search_index can return
// an index of probability 0 (its |cdf - u| < 1e-8 shortcut on a flat step, its clamp above
// the total); this never does while any p_i > 0.
__device__ __forceinline__ int select_index_nonzero(float *p, int A, float u) {
  int ind = -1, last = A - 1;        // (a row of zeros keeps the reference's clamp)
  float c = 0.0f;
  for (int i = 0; i < A; i++) {
    const float q = p[i];
    c = i ? q + c : q;
    p[i] = c;
    if (q > 0.0f) {
      last = i;
      if (ind < 0 && c >= u) ind = i;
    }
  }
  return ind >= 0 ? ind : last;
}

}  // namespace wdb
