// wdb_sa_rollout_obs_norm.cu -- the one-launch single-agent rollout (wdb_sa_rollout.cu) of a
// softmax or Gaussian policy on normalized observations: sa_rollout_kernel<kSaSoftmaxNorm> and
// <kSaGaussianNorm> of wdb_sa_rollout.cuh, in a translation unit of their own so that
// wdb_sa_rollout.cu keeps its kernels and their machine code.  wdb_single_agent_rollout
// (gaussian_head = 6 discrete, 3 continuous) checks the arguments and calls this.
#include "wdb_sa_rollout.cuh"

int sa_launch_obs_norm(void *stream, const wdb_sa_rollout *r, size_t smem) {
  if (r->env_kind >= WDB_SA_CONTINUOUS_MOUNTAIN_CAR)
    return sa_launch<kSaGaussianNorm>(stream, r, smem);
  return sa_launch<kSaSoftmaxNorm>(stream, r, smem);
}
