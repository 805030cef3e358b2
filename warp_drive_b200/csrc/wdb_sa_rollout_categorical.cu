// wdb_sa_rollout_categorical.cu -- the one-launch single-agent rollout (wdb_sa_rollout.cu) with
// C51's categorical Q head: sa_rollout_kernel<kSaCategoricalQ> of wdb_sa_rollout.cuh, in a
// translation unit of its own so that wdb_sa_rollout.cu keeps its kernels and their machine
// code.  wdb_single_agent_rollout (gaussian_head = 4) checks the arguments and calls this.
#include "wdb_sa_rollout.cuh"

int sa_launch_categorical(void *stream, const wdb_sa_rollout *r, size_t smem) {
  return sa_launch<kSaCategoricalQ>(stream, r, smem);
}
