// wdb_masked_q.cu -- DQN and C51 for envs with an action mask (include/wdb200.h,
// wdb_sample_epsilon_greedy_masked, wdb_dqn_update_masked, wdb_c51_update_masked).
//
// A Q policy's mask is a float32 row of width A beside its Q values; a non-zero entry marks a
// valid action.  Acting is epsilon-greedy over the valid actions; the update's bootstrap takes
// a* (double_q) or max_a' over the valid actions of obs' own mask, the row stored at the
// window's slot(n_step).  A row with no valid action falls back to the unmasked rule in both,
// as the masked softmax of the A2C / PPO path does: the device can neither refuse such a row
// nor wait for the host to.  With an all-ones mask every entry point gives its unmasked
// counterpart's bits.
//
// The update kernels are DQN's and C51's tile bodies (wdb_dqn_pass.cuh, wdb_c51_pass.cuh)
// instantiated with kMasked; a translation unit of their own, so the kernels of
// wdb_ddpg_update.cu and wdb_c51_update.cu keep their machine code.
#include "wdb_common.cuh"
#include "wdb_update_tiles.cuh"
#include "wdb_dqn_pass.cuh"
#include "wdb_c51_pass.cuh"

using namespace wdb;

namespace {

// ---------------------------------------------------------------------------- acting
// One thread per row, one Philox block of stream r at its offset (advanced by 1), or the words
// hook: wdb_sample_epsilon_greedy's draw and rule over the row's n_valid valid actions.  The
// row explores iff u <= eps, with the k-th valid action in ascending index order, k =
// __umulhi(y, n_valid); otherwise it takes the first maximum of Q among the valid actions.
// n_valid = A (an all-ones mask) makes both the unmasked choices.
__global__ void epsilon_greedy_masked_kernel(void *rng_state, const float *__restrict__ q,
                                             const float *__restrict__ mask,
                                             int *__restrict__ actions, long long n_rows, int A,
                                             float eps, const unsigned int *__restrict__ words) {
  const long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n_rows) return;
  unsigned long long o = 0;
  uint32_t x, y;
  if (words) {
    x = words[2 * r];
    y = words[2 * r + 1];
  } else {
    const RngHeader h = *reinterpret_cast<const RngHeader *>(rng_state);
    o = rng_offsets(rng_state)[r];
    const uint4 d = rng_draw4(h, (unsigned long long)r, o);
    x = d.x;
    y = d.y;
  }
  const float *qr = q + r * A, *mr = mask + r * A;
  int n_valid = 0;
  for (int c = 0; c < A; c++) n_valid += mr[c] != 0.0f;
  const bool all = n_valid == 0;               // no valid action: the unmasked rule
  int action = -1;
  if (u32_to_uniform(x) <= eps) {
    int k = (int)__umulhi(y, (uint32_t)(all ? A : n_valid));
    for (int c = 0; c < A && action < 0; c++)
      if (all || mr[c] != 0.0f) {
        if (k == 0) action = c;
        k--;
      }
  } else {
    float best = 0.0f;
    for (int c = 0; c < A; c++)
      if ((all || mr[c] != 0.0f) && (action < 0 || best < qr[c])) {
        best = qr[c];
        action = c;
      }
  }
  actions[r] = action;
  if (!words) rng_offsets(rng_state)[r] = o + 1;
}

// ---------------------------------------------------------------------------- update kernels
__global__ void __launch_bounds__(kThreads, 1)
dqn_masked_kernel(const float *action_mask, const __grid_constant__ wdb_dqn_update_args U,
                  const __grid_constant__ Plan Pg, float *partials, double *psums,
                  const int2 *windows) {
  dqn_tile_pass<false, true>(U, Pg, partials, psums, windows, nullptr, action_mask);
}

__global__ void __launch_bounds__(kThreads, 1)
dqn_masked_weighted_kernel(const float *action_mask, const __grid_constant__ wdb_dqn_update_args U,
                           const __grid_constant__ Plan Pg, float *partials, double *psums,
                           const int2 *windows, const float *weights) {
  dqn_tile_pass<true, true>(U, Pg, partials, psums, windows, weights, action_mask);
}

__global__ void __launch_bounds__(kThreads, 1)
c51_masked_kernel(const float *action_mask, const __grid_constant__ wdb_dqn_update_args U,
                  const __grid_constant__ Plan Pg, int N, const float *support, float dz,
                  float *partials, double *psums, const int2 *windows) {
  c51_tile_pass<false, true>(U, Pg, N, support, dz, partials, psums, windows, nullptr,
                             action_mask);
}

__global__ void __launch_bounds__(kThreads, 1)
c51_masked_prioritized_kernel(const float *action_mask,
                              const __grid_constant__ wdb_dqn_update_args U,
                              const __grid_constant__ Plan Pg, int N, const float *support,
                              float dz, float *partials, double *psums, const int2 *windows,
                              const float *weights) {
  c51_tile_pass<true, true>(U, Pg, N, support, dz, partials, psums, windows, weights,
                            action_mask);
}

}  // namespace

// ---------------------------------------------------------------------------- entry points
WDB_API int wdb_sample_epsilon_greedy_masked(void *stream, void *rng_state, const float *q_values,
                                             const float *action_mask, int *actions,
                                             long long n_rows, int n_actions, float epsilon,
                                             const unsigned int *words) {
  if (!q_values || !action_mask || !actions || n_rows <= 0 || n_actions < 1 ||
      !(epsilon >= 0.0f) || !(epsilon <= 1.0f))
    return (int)cudaErrorInvalidValue;
  if (!words && !rng_state) return (int)cudaErrorInvalidValue;
  const int block = 256;
  epsilon_greedy_masked_kernel<<<(int)((n_rows + block - 1) / block), block, 0,
                                 as_stream(stream)>>>(rng_state, q_values, action_mask, actions,
                                                      n_rows, n_actions, epsilon, words);
  return finish_launch();
}

// DQN: wdb_dqn_update_sampled's shapes and workspace
WDB_API int wdb_dqn_update_masked_supported(const wdb_dqn_update_args *u, int n_windows) {
  const wdb_replay_windows w = {nullptr, n_windows};
  Plan P;
  return qr_dqn_plan(u, 1, &w, &P) ? 1 : 0;
}
WDB_API long long wdb_dqn_update_masked_workspace_bytes(const wdb_dqn_update_args *u,
                                                        int n_windows) {
  const wdb_replay_windows w = {nullptr, n_windows};
  Plan P;
  return qr_dqn_plan(u, 1, &w, &P) ? dqn_workspace_bytes(P) : -1;
}
WDB_API int wdb_dqn_update_masked(void *stream, const wdb_dqn_update_args *u,
                                  const wdb_replay_windows *w, const float *weights,
                                  const float *action_mask) {
  Plan P;
  if (!action_mask || !qr_dqn_plan(u, 1, w, &P)) return (int)cudaErrorInvalidValue;
  static size_t configured[2] = {0, 0};
  return launch_q_pass(stream, u, P, w, weights, configured, nullptr, dqn_masked_kernel,
                       dqn_masked_weighted_kernel, action_mask, *u, P);
}

// C51: wdb_c51_update_sampled's shapes and workspace
WDB_API int wdb_c51_update_masked_supported(const wdb_dqn_update_args *u, int n_atoms,
                                            int n_windows) {
  const wdb_replay_windows w = {nullptr, n_windows};
  Plan P;
  return c51_plan(u, n_atoms, &w, &P) ? 1 : 0;
}
WDB_API long long wdb_c51_update_masked_workspace_bytes(const wdb_dqn_update_args *u,
                                                        int n_atoms, int n_windows) {
  const wdb_replay_windows w = {nullptr, n_windows};
  Plan P;
  return c51_plan(u, n_atoms, &w, &P) ? workspace_bytes(P) : -1;
}
WDB_API int wdb_c51_update_masked(void *stream, const wdb_dqn_update_args *u, int n_atoms,
                                  const float *support, float delta_z,
                                  const wdb_replay_windows *w, const float *weights,
                                  const float *action_mask) {
  Plan P;
  if (!action_mask || !c51_plan(u, n_atoms, w, &P) || !support || !(delta_z > 0.0f))
    return (int)cudaErrorInvalidValue;
  static size_t configured[2] = {0, 0};
  return launch_q_pass(stream, u, P, w, weights, configured, nullptr, c51_masked_kernel,
                       c51_masked_prioritized_kernel, action_mask, *u, P, n_atoms, support,
                       delta_z);
}
