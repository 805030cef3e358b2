// wdb_branching_q.cu -- DQN for MultiDiscrete actions by action branching (Tavakoli, Pardo &
// Kormushev 2018; include/wdb200.h, wdb_sample_epsilon_greedy_branching,
// wdb_branching_dqn_update_sampled / _prioritized).
//
// One Q head per action dimension on a shared trunk: head d is columns o_d .. o_d + A_d - 1 of
// the network's raw output, so the outputs grow with the sum of the head sizes rather than their
// product.  Acting is epsilon-greedy per head; the update bootstraps with the mean over the heads
// of each head's DQN bootstrap and regresses every head's Q(obs, a_d) on that shared return.
// With one head every entry point gives its DQN counterpart's bits.
//
// The update kernels are DQN's tile body (wdb_dqn_pass.cuh) instantiated with kBranching; a
// translation unit of its own, so the kernels of wdb_ddpg_update.cu keep their machine code.
#include "wdb_common.cuh"
#include "wdb_update_tiles.cuh"
#include "wdb_dqn_pass.cuh"
#include "wdb_sa_physics.cuh"

using namespace wdb;

namespace {

bool branches_ok(const wdb_q_branches *b) {
  if (!b || b->n_heads < 1 || b->n_heads > 16) return false;
  for (int d = 0; d < b->n_heads; d++)
    if (b->sizes[d] < 1) return false;
  return true;
}

int branches_total(const wdb_q_branches &b) {
  int A = 0;
  for (int d = 0; d < b.n_heads; d++) A += b.sizes[d];
  return A;
}

// DQN's plan with the branches' checks: sum_d A_d is the head width A
bool branching_plan(const wdb_dqn_update_args *u, const wdb_q_branches *b,
                    const wdb_replay_windows *w, Plan *p) {
  if (!u || !branches_ok(b) || branches_total(*b) != u->n_actions) return false;
  return qr_dqn_plan(u, 1, w, p);
}

// ---------------------------------------------------------------------------- acting
// One thread per row: head d takes epsilon_greedy_step (wdb_sa_physics.cuh) on its Q columns
// with the Philox block of stream r at offset o + d, or the words hook words[r][d]; the offset
// then advances by D.  At D = 1 this is epsilon_greedy_kernel (wdb_core.cu).
__global__ void epsilon_greedy_branching_kernel(void *rng_state, const float *__restrict__ q,
                                                const __grid_constant__ wdb_q_branches br,
                                                int A, int *__restrict__ actions,
                                                long long n_rows, float eps,
                                                const unsigned int *__restrict__ words) {
  const long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n_rows) return;
  const int D = br.n_heads;
  RngHeader h = {0ull, 0ull};
  unsigned long long off = 0;
  if (!words) {
    h = *reinterpret_cast<const RngHeader *>(rng_state);
    off = rng_offsets(rng_state)[r];
  }
  for (int d = 0, o = 0; d < D; o += br.sizes[d], d++)
    actions[r * D + d] = epsilon_greedy_step(q + r * A + o, br.sizes[d], eps,
                                             words ? words + 2 * (r * D + d) : nullptr, h,
                                             (unsigned long long)r, off + d);
  if (!words) rng_offsets(rng_state)[r] = off + D;
}

// ---------------------------------------------------------------------------- update kernels
__global__ void __launch_bounds__(kThreads, 1)
branching_q_pass_kernel(const __grid_constant__ wdb_q_branches br,
                        const __grid_constant__ wdb_dqn_update_args U,
                        const __grid_constant__ Plan Pg, float *partials, double *psums,
                        const int2 *windows) {
  dqn_tile_pass<false, false, true>(U, Pg, partials, psums, windows, nullptr, nullptr, &br);
}

__global__ void __launch_bounds__(kThreads, 1)
branching_q_prioritized_kernel(const __grid_constant__ wdb_q_branches br,
                               const __grid_constant__ wdb_dqn_update_args U,
                               const __grid_constant__ Plan Pg, float *partials, double *psums,
                               const int2 *windows, const float *weights) {
  dqn_tile_pass<true, false, true>(U, Pg, partials, psums, windows, weights, nullptr, &br);
}

// weights NULL: the uniform pass; else the importance-weighted one
int branching_dqn_update(void *stream, const wdb_dqn_update_args *u, const wdb_q_branches *b,
                         const wdb_replay_windows *w, const float *weights) {
  Plan P;
  if (!w || !branching_plan(u, b, w, &P)) return (int)cudaErrorInvalidValue;
  static size_t configured[2] = {0, 0};
  return launch_q_pass(stream, u, P, w, weights, configured, nullptr, branching_q_pass_kernel,
                       branching_q_prioritized_kernel, *b, *u, P);
}

}  // namespace

// ---------------------------------------------------------------------------- entry points
WDB_API int wdb_sample_epsilon_greedy_branching(void *stream, void *rng_state,
                                                const float *q_values,
                                                const wdb_q_branches *branches, int *actions,
                                                long long n_rows, float epsilon,
                                                const unsigned int *words) {
  if (!q_values || !actions || n_rows <= 0 || !branches_ok(branches) || !(epsilon >= 0.0f) ||
      !(epsilon <= 1.0f))
    return (int)cudaErrorInvalidValue;
  if (!words && !rng_state) return (int)cudaErrorInvalidValue;
  const int block = 256;
  epsilon_greedy_branching_kernel<<<(int)((n_rows + block - 1) / block), block, 0,
                                    as_stream(stream)>>>(rng_state, q_values, *branches,
                                                         branches_total(*branches), actions,
                                                         n_rows, epsilon, words);
  return finish_launch();
}

WDB_API int wdb_branching_dqn_update_sampled_supported(const wdb_dqn_update_args *u,
                                                       const wdb_q_branches *branches,
                                                       int n_windows) {
  const wdb_replay_windows w = {nullptr, n_windows};
  Plan P;
  return branching_plan(u, branches, &w, &P) ? 1 : 0;
}
WDB_API long long wdb_branching_dqn_update_sampled_workspace_bytes(
    const wdb_dqn_update_args *u, const wdb_q_branches *branches, int n_windows) {
  const wdb_replay_windows w = {nullptr, n_windows};
  Plan P;
  return branching_plan(u, branches, &w, &P) ? dqn_workspace_bytes(P) : -1;
}
WDB_API int wdb_branching_dqn_update_sampled(void *stream, const wdb_dqn_update_args *u,
                                             const wdb_q_branches *branches,
                                             const wdb_replay_windows *w) {
  return branching_dqn_update(stream, u, branches, w, nullptr);
}

// The importance-weighted pass has the uniform one's shapes and workspace
WDB_API int wdb_branching_dqn_update_prioritized_supported(const wdb_dqn_update_args *u,
                                                           const wdb_q_branches *branches,
                                                           int n_windows) {
  return wdb_branching_dqn_update_sampled_supported(u, branches, n_windows);
}
WDB_API long long wdb_branching_dqn_update_prioritized_workspace_bytes(
    const wdb_dqn_update_args *u, const wdb_q_branches *branches, int n_windows) {
  return wdb_branching_dqn_update_sampled_workspace_bytes(u, branches, n_windows);
}
WDB_API int wdb_branching_dqn_update_prioritized(void *stream, const wdb_dqn_update_args *u,
                                                 const wdb_q_branches *branches,
                                                 const wdb_replay_windows *w,
                                                 const float *weights) {
  return weights ? branching_dqn_update(stream, u, branches, w, weights)
                 : (int)cudaErrorInvalidValue;
}
