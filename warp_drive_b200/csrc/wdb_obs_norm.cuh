// wdb_obs_norm.cuh -- the float32 observation normalization that every path applies: the
// stand-alone wdb_obs_normalize launch (wdb_obs_norm.cu), which the per-step and training
// forwards call, and the one-launch single-agent rollout's normalizing kinds
// (wdb_sa_rollout.cuh).  One function, so all of them give the same bits.
#pragma once

namespace wdb {

// clamp((x - shift) * scale, -clip, clip): a rounded subtract, then a rounded multiply (no
// contraction into an fma), then the clamp.  shift and scale are the running statistics'
// float32 mean and rsqrt(var + 1e-8) (0 and 1 before the first sample).
__device__ __forceinline__ float obs_normalize(float x, float shift, float scale, float clip) {
  const float y = __fmul_rn(__fsub_rn(x, shift), scale);
  return fminf(fmaxf(y, -clip), clip);
}

}  // namespace wdb
