// wdb_sa_rollout.cu -- the WHOLE T-step rollout of a single-agent classic-control env in ONE
// launch: policy forward -> action sample -> env.step -> reward / done bookkeeping ->
// done-masked reset -> push to the training batch, T times; eight lanes share one env replica
// (the forward pass is split over them, lane 0 does the serial part of the timestep).
// Discrete kinds (CartPole, MountainCar, Acrobot; BASELINE config 3: CartPole x 10 000
// replicas) sample a softmax head; continuous kinds (ContinuousMountainCar, Pendulum: the
// DDPG configs) evaluate the actor's tanh head and add Ornstein-Uhlenbeck exploration noise,
// or (A2C / PPO with FullyConnectedGaussian) sample a Gaussian around the policy's raw mean.
//
// Replaces, per timestep, the reference's TrainerBase._generate_rollout_batch body
// (warp_drive/training/trainers/trainer_base.py:383-428): FullyConnected.forward
// (models/fully_connected.py:51-89, ~12 torch kernels), sample_actions (numba_includes/core/
// random.py / cuda_includes/core/random.cu:51-85), the env step kernel
// (example_envs/single_agent/classic_control/*/*_step_numba.py), the bookkeeping torch ops
// (trainer_base.py:514-601), reset_when_done_* (numba_includes/core/reset.py, pool_reset.py:
// 15-52) and the push-to-batch copies: ~50 launches and >= 5 host synchronisations per
// timestep there, one launch per T timesteps here.
//
// Why no tensor cores: the policies of these envs are tiny (single_cartpole.yaml: 4 -> 32 ->
// 32 -> 2, 1.3 K weights).  A 64-row wgmma tile would run K = 4 / 32 MMAs at a few percent
// of the tensor pipe and cost three launches per step; the whole network fits shared memory,
// every env's forward is evaluated in float32 by its lane group (closer to the float32 torch
// forward the update recomputes than a bf16 MMA would be), and env replicas never interact,
// so nothing has to leave the SM between timesteps.  Larger policies (H > 64) keep the
// per-step path (wgmma forward + fused step).
//
// Per timestep and env (order = the reference's): obs -> batch[t]; probs = softmax(MLP(obs));
// u ~ Philox stream `env`, one draw per call (identical to wdb_sample_actions); action via the
// reference's float32 CDF + binary search (continuous kinds: mean = scale * tanh(MLP(obs)) +
// bias, then ou_step -- the stand-alone OU sampler's own update, normal from Philox stream
// `env`); step physics = the SAME compiled device function the
// stand-alone step kernel calls (wdb_sa_physics.cuh); rewards / done -> batch[t], episodic
// sums; if done: every registered array <- its `_at_reset` row or a pool row, done = 0,
// timestep = 0 (core/reset.cu:9-75, pool_reset.py:15-52).
#include "wdb_sa_rollout.cuh"

using namespace wdb;

WDB_API int wdb_single_agent_rollout_supported(int n_hidden, const int *dims) {
  if (n_hidden < 0 || n_hidden > 3 || !dims) return 0;
  long long total = 0;
  for (int l = 0; l <= n_hidden + 1; l++)
    if (dims[l] < 1 || dims[l] > kSaMaxWidth) return 0;
  for (int l = 0; l <= n_hidden; l++) total += (long long)dims[l] * dims[l + 1] + dims[l + 1];
  return total <= kSaMaxWeights ? 1 : 0;
}

WDB_API int wdb_single_agent_rollout_categorical_supported(int n_hidden, const int *dims,
                                                           int n_atoms) {
  if (n_hidden < 0 || n_hidden > 3 || !dims || n_atoms < 2 || n_atoms > kSaMaxWidth) return 0;
  const int head = dims[n_hidden + 1];
  if (head < n_atoms || head % n_atoms != 0) return 0;
  long long total = 0;
  for (int l = 0; l <= n_hidden; l++)
    if (dims[l] < 1 || dims[l] > kSaMaxWidth) return 0;
  for (int l = 0; l <= n_hidden; l++) total += (long long)dims[l] * dims[l + 1] + dims[l + 1];
  return total <= kSaMaxWeights ? 1 : 0;
}

WDB_API int wdb_single_agent_rollout_noisy_supported(int n_hidden, const int *dims) {
  if (!wdb_single_agent_rollout_supported(n_hidden, dims)) return 0;
  const int H = dims[n_hidden], A = dims[n_hidden + 1];
  if (A > kSaGroup) return 0;                          // one output per lane
  long long total = 0;
  for (int l = 0; l <= n_hidden; l++) total += (long long)dims[l] * dims[l + 1] + dims[l + 1];
  return total + (long long)A * H + A <= kSaMaxWeights ? 1 : 0;   // mu and sigma of the head
}

// sa_rollout_kernel<kSaCategoricalQ>'s launch (wdb_sa_rollout_categorical.cu)
int sa_launch_categorical(void *stream, const wdb_sa_rollout *r, size_t smem);
// sa_rollout_kernel<kSaNoisyQ>'s launch (wdb_sa_rollout_noisy.cu)
int sa_launch_noisy(void *stream, const wdb_sa_rollout *r, size_t smem);
// sa_rollout_kernel<kSaSoftmaxNorm / kSaGaussianNorm>'s launch (wdb_sa_rollout_obs_norm.cu)
int sa_launch_obs_norm(void *stream, const wdb_sa_rollout *r, size_t smem);

WDB_API int wdb_single_agent_rollout(void *stream, const wdb_sa_rollout *r) {
  if (!r) return (int)cudaErrorInvalidValue;
  const int rc = sa_check_env_arrays(r->env_kind, r->n_envs, r->state, r->sampled_actions,
                                     r->done, r->rewards, r->observations, r->env_timestep);
  if (rc != cudaSuccess) return rc;
  const bool continuous = r->env_kind >= WDB_SA_CONTINUOUS_MOUNTAIN_CAR;
  const bool squashed = continuous && r->gaussian_head == 2;
  // the softmax (6) and Gaussian (3) heads on normalized observations
  const bool normalized = continuous ? r->gaussian_head == 3 : r->gaussian_head == 6;
  const bool gaussian = continuous && (r->gaussian_head == 1 || normalized);
  const bool eps_greedy = !continuous && r->gaussian_head == 3;
  const bool categorical = !continuous && r->gaussian_head == 4;
  const bool noisy = !continuous && r->gaussian_head == 5;
  if (r->n_steps <= 0) return (int)cudaErrorInvalidValue;
  // the categorical head: A blocks of N atoms, A = the kind's action count
  const int n_atoms = categorical ? r->dims[r->n_hidden + 1] / kSaNActions[r->env_kind] : 1;
  if (categorical ? !wdb_single_agent_rollout_categorical_supported(r->n_hidden, r->dims, n_atoms)
      : noisy     ? !wdb_single_agent_rollout_noisy_supported(r->n_hidden, r->dims)
                  : !wdb_single_agent_rollout_supported(r->n_hidden, r->dims))
    return (int)cudaErrorInvalidValue;
  for (int l = 0; l <= r->n_hidden; l++)
    if (!r->w[l] || !r->b[l]) return (int)cudaErrorInvalidValue;
  if (continuous && (r->gaussian_head < 0 || r->gaussian_head > 3))
    return (int)cudaErrorInvalidValue;
  if (normalized && !r->log_std) return (int)cudaErrorInvalidValue;
  if (squashed || gaussian) {
    // log_std, and a normal source unless the deterministic action draws nothing
    if (!r->log_std || (!r->use_argmax && !r->normals && !r->rng_state))
      return (int)cudaErrorInvalidValue;
  } else if (continuous) {
    // the OU state and a normal source unless the bypass (scale < 1e-8) draws nothing
    if (!(r->ou_scale < 1.0e-8f) && (!r->ou_state || (!r->normals && !r->rng_state)))
      return (int)cudaErrorInvalidValue;
  } else if (eps_greedy || categorical || noisy) {
    // epsilon on the device; one Philox draw per step whatever it is; no uniforms hook
    if (!r->log_std || !r->rng_state || r->uniforms) return (int)cudaErrorInvalidValue;
  } else if (!r->use_argmax && !r->uniforms && !r->rng_state) {
    return (int)cudaErrorInvalidValue;
  }
  // the observation feeds the first layer, and the head is one logit per discrete action
  // (one tanh output for the continuous kinds): a wider head would step the env with actions
  // it does not have; the squashed head is [mu, log-std] of the one action, the categorical
  // head N atoms per action
  const int head = kSaNActions[r->env_kind] * (squashed ? 2 : n_atoms);
  if (r->state_dim != kSaStateDim[r->env_kind] || r->dims[0] != kSaObsDim[r->env_kind] ||
      r->dims[r->n_hidden + 1] != head)
    return (int)cudaErrorInvalidValue;
  if (r->reset_done_envs && r->n_reset_arrays > 0 && !r->reset_table)
    return (int)cudaErrorInvalidValue;
  long long total = 0;
  for (int l = 0; l <= r->n_hidden; l++)
    total += (long long)r->dims[l] * r->dims[l + 1] + r->dims[l + 1];
  const size_t smem = ((size_t)total + (size_t)kSaEnvsPerCta * 2 * kSaPitch) * sizeof(float);
  if (normalized) return sa_launch_obs_norm(stream, r, smem);
  if (squashed) return sa_launch<kSaSquashed>(stream, r, smem);
  if (gaussian) return sa_launch<kSaGaussian>(stream, r, smem);
  if (eps_greedy) return sa_launch<kSaEpsGreedy>(stream, r, smem);
  // (and each env's Q row, and the support)
  if (noisy) {                         // (and the head's sigma_W, sigma_b)
    const int H = r->dims[r->n_hidden], A = r->dims[r->n_hidden + 1];
    return sa_launch_noisy(stream, r, smem + (size_t)(A * H + A) * sizeof(float));
  }
  if (categorical)
    return sa_launch_categorical(
        stream, r, smem + ((size_t)kSaEnvsPerCta * kSaPitch + kSaMaxWidth) * sizeof(float));
  return continuous ? sa_launch<kSaTanhOu>(stream, r, smem) : sa_launch<kSaSoftmax>(stream, r, smem);
}
