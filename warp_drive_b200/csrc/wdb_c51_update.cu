// wdb_c51_update.cu -- one categorical DQN update (C51; Bellemare, Dabney & Munos 2017) of one
// policy over B sampled replay windows, in two launches: a tile kernel and the fixed-order
// reduction of its per-CTA partials (include/wdb200.h, wdb_c51_update_sampled).
//
// The networks: DQN's trunk (hidden Linear + ReLU layers) and a raw head of A * N atom logits,
// row a * N + j of the head the logit of atom j of action a.  A head wider than one tile row
// (64 columns: 102 for CartPole, 153 for MountainCar and Acrobot at N = 51) is held and run as A
// blocks of N <= 64 rows, block a the contiguous head rows [a N, (a + 1) N), each laid out in
// shared memory as a Linear of its own (N weight rows, then N biases).  Per tile of kRows
// sampled windows:
//   - the online trunk on obs (its hidden outputs kept for the backward) and the chooser's
//     (online with double_q, else the target) on obs';
//   - every block of the chooser at obs', each reduced to its expectation; a* the first argmax;
//   - the target's trunk on obs' (double_q) and, per row, its block a* (the gathered forward:
//     each row through its own block): p' = softmax over the atoms;
//   - per row, on its 16 threads: Tz_j = DQN's n-step recursion on z_j, clamped to the support;
//     the N x N projection pairs (thread k owns the atoms i = k, k + 16, ... and sums over j in
//     order); the online block a at obs (gathered) and its log-softmax; the cross-entropy and
//     its logit gradient;
//   - the head gradient block by block (each block's rows masked to the windows of that
//     action), d psi through the gathered blocks, then back through the trunk.
// Every sum runs in a fixed order and the partials are reduced in CTA order: an update is
// bit-reproducible.  Its own translation unit, on the primitives of wdb_update_tiles.cuh, so
// the kernels of wdb_ddpg_update.cu and wdb_iqn_update.cu keep their machine code.  The tile
// body, its head-block primitives and the plan are in wdb_c51_pass.cuh, which the action-masked
// pass (wdb_masked_q.cu) shares.
#include "wdb_common.cuh"
#include "wdb_update_tiles.cuh"
#include "wdb_c51_pass.cuh"                // C51's tile body and plan

using namespace wdb;

namespace {

__global__ void __launch_bounds__(kThreads, 1)
c51_kernel(const __grid_constant__ wdb_dqn_update_args U, const __grid_constant__ Plan Pg, int N,
           const float *support, float dz, float *partials, double *psums, const int2 *windows) {
  c51_tile_pass<false>(U, Pg, N, support, dz, partials, psums, windows, nullptr);
}

__global__ void __launch_bounds__(kThreads, 1)
c51_prioritized_kernel(const __grid_constant__ wdb_dqn_update_args U,
                       const __grid_constant__ Plan Pg, int N, const float *support, float dz,
                       float *partials, double *psums, const int2 *windows,
                       const float *weights) {
  c51_tile_pass<true>(U, Pg, N, support, dz, partials, psums, windows, weights);
}

// weights NULL: the uniform-replay kernel; else the importance-weighted one.
int c51_update_sampled(void *stream, const wdb_dqn_update_args *u, int N, const float *support,
                       float dz, const wdb_replay_windows *w, const float *weights) {
  Plan P;
  if (!c51_plan(u, N, w, &P) || !support || !(dz > 0.0f)) return (int)cudaErrorInvalidValue;
  static size_t configured[2] = {0, 0};
  return launch_q_pass(stream, u, P, w, weights, configured, nullptr, c51_kernel,
                       c51_prioritized_kernel, *u, P, N, support, dz);
}

}  // namespace

// ---------------------------------------------------------------------------- entry points
// C51: DQN's argument struct, the number of atoms, the support and its spacing
WDB_API int wdb_c51_update_sampled_supported(const wdb_dqn_update_args *u, int n_atoms,
                                             int n_windows) {
  const wdb_replay_windows w = {nullptr, n_windows};
  Plan P;
  return c51_plan(u, n_atoms, &w, &P) ? 1 : 0;
}
WDB_API long long wdb_c51_update_sampled_workspace_bytes(const wdb_dqn_update_args *u,
                                                         int n_atoms, int n_windows) {
  const wdb_replay_windows w = {nullptr, n_windows};
  Plan P;
  return c51_plan(u, n_atoms, &w, &P) ? workspace_bytes(P) : -1;
}
WDB_API int wdb_c51_update_sampled(void *stream, const wdb_dqn_update_args *u, int n_atoms,
                                   const float *support, float delta_z,
                                   const wdb_replay_windows *w, const float *weights) {
  return c51_update_sampled(stream, u, n_atoms, support, delta_z, w, weights);
}
