// wdb_sa_rollout_noisy.cu -- the one-launch single-agent rollout (wdb_sa_rollout.cu) with a
// noisy DQN head: sa_rollout_kernel<kSaNoisyQ> of wdb_sa_rollout.cuh, in a translation unit of
// its own so that wdb_sa_rollout.cu keeps its kernels and their machine code.
// wdb_single_agent_rollout (gaussian_head = 5) checks the arguments and calls this.
#include "wdb_sa_rollout.cuh"

int sa_launch_noisy(void *stream, const wdb_sa_rollout *r, size_t smem) {
  return sa_launch<kSaNoisyQ>(stream, r, smem);
}
