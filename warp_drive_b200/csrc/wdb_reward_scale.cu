// wdb_reward_scale.cu -- the running discounted return that reward scaling divides by
// (include/wdb200.h, wdb_discounted_return_scan).
//
// One thread per (env, agent) row walks the batch forward in time from the row's carried
// return: ret = gamma * carry + r_t, returns[t] = ret, then the carry restarts at 0 when the
// env's episode ended at t (SB3 VecNormalize's order).  The multiply and the add are the
// explicit _rn intrinsics, so no FMA is contracted and a float32 restatement on the host gives
// the same bits.  Each step's loads and stores are unit-stride across the rows.  The moments of
// the returns and the scaling reuse wdb_obs_moments_* and wdb_obs_normalize with F = 1.
#include "wdb_common.cuh"

using namespace wdb;

namespace {

constexpr int kThreads = 128;
constexpr int kAhead = 8;   // steps whose loads are in flight ahead of the serial chain

__global__ void __launch_bounds__(kThreads)
discounted_return_scan_kernel(const float *__restrict__ rewards, const int *__restrict__ done,
                              int T, int E, int Np, float gamma, float *__restrict__ carry,
                              float *__restrict__ returns) {
  const long long per_t = (long long)E * Np;
  const long long i = (long long)blockIdx.x * kThreads + threadIdx.x;
  if (i >= per_t) return;
  const long long env = i / Np;
  float c = carry[i];
  int t = 0;
  for (; t + kAhead <= T; t += kAhead) {
    float r[kAhead];
    int d[kAhead];
#pragma unroll
    for (int j = 0; j < kAhead; j++) {
      r[j] = rewards[(long long)(t + j) * per_t + i];
      d[j] = done[(long long)(t + j) * E + env];
    }
#pragma unroll
    for (int j = 0; j < kAhead; j++) {
      const float ret = __fadd_rn(__fmul_rn(gamma, c), r[j]);
      returns[(long long)(t + j) * per_t + i] = ret;
      c = d[j] > 0 ? 0.0f : ret;
    }
  }
  for (; t < T; t++) {
    const float ret = __fadd_rn(__fmul_rn(gamma, c), rewards[(long long)t * per_t + i]);
    returns[(long long)t * per_t + i] = ret;
    c = done[(long long)t * E + env] > 0 ? 0.0f : ret;
  }
  carry[i] = c;
}

}  // namespace

WDB_API int wdb_discounted_return_scan(void *stream, const float *rewards, const int *done,
                                       int T, int n_envs, int n_agents, float gamma,
                                       float *carry, float *returns) {
  if (!rewards || !done || !carry || !returns || T < 1 || n_envs < 1 || n_agents < 1)
    return (int)cudaErrorInvalidValue;
  const long long rows = (long long)n_envs * n_agents;
  const long long blocks = (rows + kThreads - 1) / kThreads;
  if (blocks > 0x7fffffffLL) return (int)cudaErrorInvalidValue;
  discounted_return_scan_kernel<<<(unsigned)blocks, kThreads, 0, as_stream(stream)>>>(
      rewards, done, T, n_envs, n_agents, gamma, carry, returns);
  return finish_launch();
}
