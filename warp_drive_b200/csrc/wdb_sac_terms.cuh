// wdb_sac_terms.cuh -- the per-row pieces of the SAC-family replay passes: the n-step return of
// a sampled window (DDPG, TD3, SAC in wdb_ddpg_update.cu; TQC in wdb_tqc.cu) and one dimension of
// the tanh-squashed Gaussian (SAC, TQC).  Each translation unit gets its own copy (anonymous
// namespace), as with wdb_update_tiles.cuh.
#pragma once

#include "wdb_update_tiles.cuh"

namespace {

// The n-step return of sampled window w from its bootstrap value qt: the recursion of a
// regular window of the ring in the same float32 operations, for every SAC-family
// argument struct (DDPG, TD3, SAC, TQC).
template <class Args>
__device__ __forceinline__ float sampled_return(const Args &U, const Plan &P,
                                                const SampledRows &rows, const Row &w, float qt) {
  const int ns = U.n_step;
  const long long EN = P.EN, E = U.n_envs, n = w.n, env = n / U.n_agents;
  float ret = qt;
  for (int j = ns - 1; j >= 0; j--) {
    const int pk = rows.slot(w, j);
    const float dk = (float)U.done[(long long)pk * E + env];
    const float rk = U.rewards[(long long)pk * EN + n];
    ret = __fadd_rn(__fmul_rn(__fmul_rn(__fsub_rn(1.0f, dk), U.gamma), ret), rk);
  }
  return ret;
}

// One action dimension of the squashed Gaussian at head row z (mu in column c, the raw log-std
// in column A + c) and standard normal eps: u = mu + exp(log_std) eps and the dimension's
// log-prob term -eps^2 / 2 - log_std - log(2 pi) / 2 - 2 (log 2 - u - softplus(-2 u))
// (softplus as torch's, threshold 20).
struct SquashedDim {
  float sigma, u, y, term;
  bool in_range;                     // the raw log-std lies in [lo, hi]: the clamp passes d/draw
};

__device__ __forceinline__ SquashedDim squashed_dim(const float *z, int A, int c, float eps,
                                                    float lo, float hi) {
  const float raw = z[A + c];
  SquashedDim s;
  s.in_range = raw >= lo && raw <= hi;
  const float ls = fminf(fmaxf(raw, lo), hi);
  s.sigma = expf(ls);
  s.u = fmaf(s.sigma, eps, z[c]);
  s.y = tanhf(s.u);
  const float x = -2.0f * s.u;
  const float sp = x > 20.0f ? x : log1pf(expf(x));
  const float corr = 2.0f * (0.69314718055994531f - s.u - sp);
  s.term = -0.5f * eps * eps - ls - 0.91893853320467274f - corr;
  return s;
}

}  // namespace
