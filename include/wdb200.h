/*
 * wdb200.h -- C ABI of libwdb200.so, the H100-native (sm_90a) rollout kernels that
 * replace WarpDrive's JIT-compiled CUDA module.
 *
 * Boundary being replaced (reference = salesforce/warp-drive v2.7.1): the reference
 * looks kernels up BY NAME in a pycuda module and launches them with positional
 * arguments (warp_drive/managers/pycuda_managers/pycuda_function_manager.py:319-388,
 * `get_function(name)(*args, block=, grid=)`).  Each entry point below takes the same
 * arguments, in the same order, as the reference kernel it replaces, with three
 * changes: (1) a leading `stream` (cudaStream_t as void*; NULL = legacy default
 * stream), (2) the compile-time constants wkNumberEnvs / wkNumberAgents /
 * wkBlocksPerEnv (warp_drive/cuda_includes/template_env_config.h:19-21) become run-time
 * arguments, (3) `bool` kernel parameters become int32 (the reference passes np.int32
 * into `bool` params, SURVEY.md section 8 "Python-side arg passing").
 *
 * Conventions
 *   - every function returns a cudaError_t as int (0 == cudaSuccess) and never throws;
 *     wdb_error_string() turns it into text.  Launches are asynchronous on `stream`.
 *   - all buffers are caller-owned device memory (torch CUDA tensors), row-major,
 *     C-contiguous, 32-bit elements.  State arrays are updated in place
 *     (warp_drive/env_wrapper.py:347-352).
 *   - the library allocates nothing; RNG state is a caller-provided blob of
 *     wdb_rng_state_bytes(n_streams) bytes.
 *   - one host thread per process, one process per GPU.
 */
#ifndef WDB200_H_
#define WDB200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define WDB_ABI_VERSION 1

int wdb_abi_version(void);
const char *wdb_error_string(int err);
/* number of kernel launches issued through this library since load (bench.py's
 * `gpu_launches` evidence) */
long long wdb_launch_count(void);

/* Tuning / A-B switches (results are identical either way).  "tc_history": use last step's
 * neighbour lists as a distance threshold in the tag_continuous k-nearest search (1, default)
 * or always run the full sorting network (0).  "tc_force_exact": resolve every agent's
 * neighbours with the reference's literal selection (1) instead of only the ambiguous ones
 * (0, default).  "tc_cta_threads": thread budget of one
 * tag_continuous CTA (32..320, default 320); a CTA takes floor(budget / agents) envs.
 * "mlp_max_ctas": persistent CTAs (= SMs) the following wdb_mlp_policy_forward launches may
 * use (0 = all): two policies' forwards can then run concurrently on disjoint SMs. */
int wdb_set_option(const char *name, int value);

/* ------------------------------------------------------------------ RNG ------ */
/* Replaces init_random / free_random (warp_drive/cuda_includes/core/random.cu:14-31):
 * the reference heap-allocates one XORWOW curandState per (env, agent) thread; here the
 * state is a flat caller-owned blob: {u64 seed, u64 n_streams, u64 offset[n_streams]}
 * driving a counter-based Philox4x32-10 (key = seed, counter = {offset, stream}). */
long long wdb_rng_state_bytes(long long n_streams);
int wdb_rng_init(void *stream, void *rng_state, long long n_streams,
                 unsigned long long seed);

/* Test hook: out[4*i .. 4*i+3] = the next Philox block of stream i (advances every
 * stream's offset by one) -- lets tests pin the device RNG against the scalar oracle. */
int wdb_rng_draw_u32x4(void *stream, void *rng_state, unsigned int *out,
                       long long n_streams);

/* Replaces sample_actions (random.cu:51-85; launched from PyCUDASampler.sample,
 * pycuda_function_manager.py:532-572).  probs [n_envs, n_agents, n_actions] f32.
 * actions [n_envs, n_agents, 1] i32.  cum_distr [n_envs, n_agents, n_actions] f32 or
 * NULL (the reference always materialises it; it is scratch).  actions_combined
 * (optional) receives the same index at [pos * combined_stride + combined_offset] --
 * the reference does that with a separate torch copy (trainer_base.py:507-512).
 * uniforms (optional, test hook): if non-NULL the draw p is read from uniforms[pos]
 * instead of the RNG, which makes the index selection parity-testable. */
int wdb_sample_actions(void *stream, void *rng_state, const float *probs, int *actions,
                       float *cum_distr, int n_envs, int n_agents, int n_actions,
                       int use_argmax, int *actions_combined, int combined_stride,
                       int combined_offset, const float *uniforms);
/* The same sampler with a selection that never returns a zero-probability index (for
 * policies whose actions are masked): the first index i with p_i > 0 and cdf_i >= u; when u
 * lies above the float32 total, the last index with p_i > 0.  The reference's search
 * (wdb_sample_actions) can land on a flat CDF step or clamp to the last index, both of
 * which may carry probability 0.  Same arguments, same RNG draws, same cum_distr. */
int wdb_sample_actions_nonzero(void *stream, void *rng_state, const float *probs, int *actions,
                               float *cum_distr, int n_envs, int n_agents, int n_actions,
                               int use_argmax, int *actions_combined, int combined_stride,
                               int combined_offset, const float *uniforms);

/* Replaces the numba-only sample_ou_process (warp_drive/numba_includes/core/random.py:
 * 74-105): ou = (1-damping)*ou + stddev*N(0,1); action = mean + scale*ou.
 * normals (optional, test hook) replaces the N(0,1) draw. */
int wdb_sample_ou_process(void *stream, void *rng_state, const float *mean,
                          float *actions, float *ou_state, int n_envs, int n_agents,
                          float damping, float stddev, float scale,
                          const float *normals);

/* Diagonal Gaussian policy with a state-independent log-std (FullyConnectedGaussian):
 *   actions[r, k] = fmaf(expf(log_std[k]), n, mean[r, k]),  n ~ N(0, 1).
 * mean / actions [n_rows, action_dim] f32, log_std [action_dim].  Row r draws from Philox stream
 * r at its own offset (as wdb_sample_ou_process): dims 2j and 2j+1 come from the j-th draw,
 * u32x2_to_normal(x, y) and u32x2_to_normal(z, w), so one dimension is exactly the OU
 * sampler's draw.  use_argmax: actions = mean, nothing drawn, offsets untouched (the
 * evaluator's deterministic action).  normals (optional, test hook) [n_rows, action_dim]
 * replaces the draws.  The sample is written raw, NOT clipped to the action space: bounds are
 * the env's business (Pendulum and ContinuousMountainCar clip inside their physics), so the
 * update's log-prob is taken at exactly the action the env received. */
int wdb_sample_gaussian(void *stream, void *rng_state, const float *mean, const float *log_std,
                        float *actions, long long n_rows, int action_dim, int use_argmax,
                        const float *normals);

/* Tanh-squashed Gaussian policy (SAC's actor): row r of `head` [n_rows, 2A] holds the mean mu
 * (columns [0, A)) and the raw log-std (columns [A, 2A)), which is clamped to
 * [log_std_min, log_std_max]; with u = mu + exp(log_std) * n,
 *   actions[r][k] = action_scale * tanh(u_k) + action_bias,
 * n drawn as wdb_sample_gaussian draws (row r on Philox stream r, two dimensions per draw) or
 * read from `normals` [n_rows, A] (test hook).  use_argmax: u = mu, nothing drawn. */
int wdb_sample_squashed_gaussian(void *stream, void *rng_state, const float *head,
                                 float *actions, long long n_rows, int action_dim,
                                 float action_scale, float action_bias, float log_std_min,
                                 float log_std_max, int use_argmax, const float *normals);

/* Epsilon-greedy over Q values (DQN): row r of `q_values` [n_rows, n_actions] takes ONE
 * Philox4x32-10 block (x, y, z, w) on stream r at its offset, which then advances by 1; or the
 * words (x, y) = words[r] [n_rows][2] (test hook; no RNG state read or advanced).  With u =
 * x * 2^-32 + 2^-33 in float32 (the (0, 1] uniform of wdb_sample_actions), the row explores iff
 * u <= epsilon, with action = high word of y * n_actions; otherwise the action is the first
 * index of the maximum Q value.  cudaErrorInvalidValue unless 0 <= epsilon <= 1. */
int wdb_sample_epsilon_greedy(void *stream, void *rng_state, const float *q_values,
                              int *actions, long long n_rows, int n_actions, float epsilon,
                              const unsigned int *words);

/* wdb_sample_epsilon_greedy over the valid actions of action_mask [n_rows, n_actions] (float32,
 * non-zero = valid): the same draw (one Philox block per row on stream r, the offset advanced by
 * 1, or the words hook) and the same u.  With n_valid the row's valid actions, the row explores
 * iff u <= epsilon, with the k-th valid action in ascending index order, k = high word of
 * y * n_valid; otherwise it takes the first index of the maximum Q value among the valid
 * actions.  A row with no valid action takes wdb_sample_epsilon_greedy's action (the device
 * can neither refuse it nor report it without a host wait).  An all-ones mask gives
 * wdb_sample_epsilon_greedy's actions and offsets bit for bit.  One launch.
 * cudaErrorInvalidValue unless 0 <= epsilon <= 1, or if action_mask is NULL. */
int wdb_sample_epsilon_greedy_masked(void *stream, void *rng_state, const float *q_values,
                                     const float *action_mask, int *actions, long long n_rows,
                                     int n_actions, float epsilon, const unsigned int *words);

/* ------------------------------------------------------------------ reset ---- */
/* Replaces reset_in_{float,int}_when_done_{2d,3d} + undo_done_flag_and_reset_timestep
 * (warp_drive/cuda_includes/core/reset.cu:9-75; one launch per registered array in
 * PyCUDAEnvironmentReset.reset_when_done_deterministic, pycuda_function_manager.py:
 * 668-753) and the numba-only reset_when_done_{1,2,3}d_from_pool
 * (numba_includes/core/pool_reset.py:15-52) with ONE launch over a device-resident
 * descriptor table. */
typedef struct wdb_reset_desc {
  void *dst;                /* data[env]            */
  const void *ref;          /* data_at_reset[env] or pool[row]                      */
  long long bytes_per_env;  /* multiple of 4                                        */
  long long pool_rows;      /* 0: deterministic (ref indexed by env); >0: pool size */
} wdb_reset_desc;

int wdb_reset_when_done(void *stream, const wdb_reset_desc *table_dev, int n_arrays,
                        int *done, int *timestep, int n_envs, int force_reset,
                        int undo_done_and_timestep, void *pool_rng_state);

/* ------------------------------------------------------------------ log ------ */
/* Replace reset_log_mask / update_log_mask / log_one_step_in_{float,int}
 * (warp_drive/cuda_includes/core/log.cu:11-62). */
int wdb_reset_log_mask(void *stream, int *log_mask, int episode_length);
int wdb_update_log_mask(void *stream, int *log_mask, int timestep, int episode_length);
int wdb_log_one_step(void *stream, void *log, const void *data, int n_agents,
                     int feature_dim, int timestep, int episode_length, int env_id);

/* ------------------------------------------------------------------ envs ----- */
/* Replaces testkernel (example_envs/dummy_env/test_step.cu:9-45). */
int wdb_testkernel(void *stream, int n_envs, int n_agents, float *x, int *y, int *done,
                   int *actions, float multiplier, int target, int step,
                   int episode_length);

/* Replaces CudaTagGridWorldStep (example_envs/tag_gridworld/
 * tag_gridworld_step_pycuda.cu:112-251; argument order of tag_gridworld.py:353-368).
 * index_to_action: device int[10], the reference's __constant__ kIndexToActionArr. */
int wdb_tag_gridworld_step(void *stream, int n_envs, int n_agents, int *loc_x,
                           int *loc_y, const int *actions, int *done, float *rewards,
                           float *obs, float wall_hit_penalty,
                           float tag_reward_for_tagger, float tag_penalty_for_runner,
                           float step_cost_for_tagger, int use_full_observation,
                           int world_boundary, int *env_timestep, int episode_length,
                           const int *index_to_action);

/* Replaces CudaTagContinuousStep (example_envs/tag_continuous/
 * tag_continuous_step_pycuda.cu:351-520; argument order of tag_continuous.py:806-840).
 * neighbor_distances / neighbor_ids_sorted_by_distance are the reference's O(N^2)
 * global scratch; they may be NULL (the native kernel keeps the sweep on chip).
 * stats (optional, device int[4]): [0] += agents that took the exact tie-resolution
 * path, [1] += tags, [2] += agents whose threshold scan had no usable candidate list
 * (full sorting network), [3] += agents whose candidate list overflowed (cluster kernel:
 * sorting network over the x-window only). */
int wdb_tag_continuous_step(
    void *stream, int n_envs, int n_agents, int blocks_per_env, float *loc_x,
    float *loc_y, float *speed, float *direction, float *acceleration,
    const int *agent_types, float *edge_hit_reward_penalty, float edge_hit_penalty,
    float grid_length, const float *acceleration_actions, const float *turn_actions,
    float max_speed, int num_other_agents_observed, const float *skill_levels,
    int runner_exits_game_after_tagged, int *still_in_the_game,
    int use_full_observation, float *obs, const int *action_indices,
    float *neighbor_distances, int *neighbor_ids_sorted_by_distance,
    int *nearest_neighbor_ids, float *rewards, const float *step_rewards,
    int *num_runners, float distance_margin_for_reward, float tag_reward_for_tagger,
    float tag_penalty_for_runner, float end_of_game_reward_for_runner, int *done,
    int *env_timestep, int episode_length, int *stats);

/* ------------------------------------------------------------ fused rollout step -- */
/* ONE launch per rollout timestep of tag_continuous:
 *   sample both action heads from the policies' probabilities (sample_actions x2,
 *   core/random.cu:51-85) -> CudaTagContinuousStep -> push actions / rewards / done to the
 *   training batch slots and update the episodic sums (trainer_base.py:437-601) ->
 *   write the new observations per policy for the next forward pass
 *   (model_base.py:181-200) -> done-masked reset of every registered array + undo of
 *   done/timestep (core/reset.cu:9-75; function_manager.py:256-273).
 * The reference issues ~50 launches and >= 5 host syncs for the same work. */
typedef struct wdb_tc_env {          /* the arguments of wdb_tag_continuous_step */
  int n_envs, n_agents;
  float *loc_x, *loc_y, *speed, *direction, *acceleration;
  const int *agent_types;
  float *edge_hit_reward_penalty;
  float edge_hit_penalty, grid_length;
  const float *acceleration_actions, *turn_actions;
  float max_speed;
  int num_other_agents_observed;
  const float *skill_levels;
  int runner_exits_game_after_tagged;
  int *still_in_the_game;
  int use_full_observation;
  float *obs;                        /* [E, N, F]; may be NULL when obs_next is used */
  float *neighbor_distances;         /* optional scratch */
  int *neighbor_ids_sorted_by_distance;
  int *nearest_neighbor_ids;
  float *rewards;
  const float *step_rewards;
  int *num_runners;
  float distance_margin_for_reward, tag_reward_for_tagger, tag_penalty_for_runner,
      end_of_game_reward_for_runner;
  int *done, *env_timestep;
  int episode_length;
  int *stats;
  int blocks_per_env;                /* <= 1: env replicas packed into CTAs; > 1: one env per
                                      * cluster of that many CTAs (as wdb_tag_continuous_step) */
} wdb_tc_env;

typedef struct wdb_tc_policy_io {    /* per policy; agents of a policy are [E, Np, ...] */
  int n_agents;                      /* Np */
  const float *probs0, *probs1;      /* [E, Np, A0], [E, Np, A1] from the forward pass */
  int *actions_batch;                /* [E, Np, 2]  slot t of sampled_actions_batch_p, or NULL */
  float *rewards_batch;              /* [E, Np]     slot t of rewards_batch_p, or NULL */
  float *obs_next;                   /* [E, Np, F]  where the next forward reads, or NULL */
  float *reward_running_sum;         /* [E, Np] or NULL */
  float *episodic_reward_sum;        /* scalar or NULL */
  void *obs_next_tiles;              /* optional bf16 copy of obs_next in the A-operand tile
                                      * layout of wdb_mlp_policy_forward_tiles
                                      * (wdb_mlp_obs_tiles_bytes bytes, 16-byte aligned), or NULL */
} wdb_tc_policy_io;

typedef struct wdb_tc_rollout {
  void *rng_state;
  const float *uniforms;             /* test hook [E, N, 2]; NULL = device RNG */
  int n_policies, n_actions0, n_actions1;
  const int *agent_policy;           /* [N] policy index of every agent */
  const int *agent_slot;             /* [N] index of the agent inside its policy */
  wdb_tc_policy_io policy[4];
  int *sampled_actions;              /* [E, N, 2] or NULL */
  int *sampled_actions_0, *sampled_actions_1;   /* [E, N, 1] or NULL */
  int *done_batch;                   /* [E] slot t of done_flags_batch, or NULL */
  int *step_running_sum;             /* [E] or NULL */
  unsigned long long *episodic_step_sum, *num_completed_episodes;   /* scalars or NULL */
  const wdb_reset_desc *reset_table; /* device table of the arrays to restore */
  int n_reset_arrays;
  const float *obs_at_reset;         /* [E, N, F]: source of obs_next for envs that reset */
  int reset_done_envs;               /* 0: leave done envs alone (done stays set) */
  int launch_after_forward;          /* 1: the kernel launched just before this one on `stream`
                                      * is this step's policy forward (and the one before that
                                      * the previous env step): with the "pdl" option on, the
                                      * launch is programmatically dependent on it -- the state
                                      * prologue overlaps the forward's tail, the probabilities
                                      * are read after griddepcontrol.wait.  0: plain launch. */
  int actions_in;                    /* 1: the actions were already sampled (by
                                      * wdb_mlp_policy_forward_sampled) into every policy's
                                      * actions_batch, which is then required and only read;
                                      * probs0 / probs1 and the RNG are not used.  Only the packed
                                      * kernel of up to 320 threads per CTA takes this mode
                                      * (wdb_tag_continuous_rollout_supported reads this field). */
  int env_begin, env_count;          /* step envs [env_begin, env_begin + env_count) only (0, 0:
                                      * all); every array is still the whole [E, ...] one,
                                      * addressed by global env and agent index.  Only the packed
                                      * kernel takes a proper subrange. */
} wdb_tc_rollout;

int wdb_tag_continuous_rollout_step(void *stream, const wdb_tc_env *env,
                                    const wdb_tc_rollout *rollout);

/* Whether wdb_tag_continuous_rollout_step can run this env and rollout shape: 0, or the code
 * it would return once every pointer of `rollout` is valid, with obs_next written for every
 * policy and obs_next_tiles for every policy iff with_obs_tiles.  Only the shape fields of
 * `rollout` are read (n_policies, n_actions0/1, policy[].n_agents, the reset fields); `env`
 * is read as the step reads it.  No pointer is dereferenced and no CUDA call is made.  The
 * verdict depends on the wdb_set_option switches at the time of the call. */
int wdb_tag_continuous_rollout_supported(const wdb_tc_env *env, const wdb_tc_rollout *rollout,
                                         int with_obs_tiles);

/* Replaces NumbaClassicControlCartPoleEnvStep (example_envs/single_agent/
 * classic_control/cartpole/cartpole_step_numba.py:6-83; argument order of
 * cartpole.py:105-122). */
int wdb_cartpole_step(void *stream, int n_envs, float *state, const int *action,
                      int *done, float *reward, float *obs, float gravity,
                      float masspole, float total_mass, float length,
                      float polemass_length, float force_mag, float tau,
                      float theta_threshold_radians, float x_threshold,
                      int *env_timestep, int episode_length);

/* ------------------------------------------------- classic control (SURVEY 8 f2) ---- */
/* The four remaining single-agent envs of example_envs/single_agent/classic_control/.
 * The reference has them only as numba kernels launched as one 1-thread block per env;
 * argument order below = the kernel signatures (and the `args` lists of the env classes'
 * step()), with n_envs made explicit.  state/obs rows are [n_envs, 1, k] float32. */

/* Replaces NumbaClassicControlMountainCarEnvStep (mountain_car/mountain_car_step_numba.py:
 * 14-70; args of mountain_car.py:104-119).  state/obs k = 2, action int32 [E,1,1].
 * done = 1 at the episode end, 2 when the goal is reached (as the reference). */
int wdb_mountain_car_step(void *stream, int n_envs, float *state, const int *action,
                          int *done, float *reward, float *obs, float min_position,
                          float max_position, float max_speed, float goal_position,
                          float goal_velocity, float force, float gravity,
                          int *env_timestep, int episode_length);

/* Replaces NumbaClassicControlContinuousMountainCarEnvStep (continuous_mountain_car/
 * continuous_mountain_car_step_numba.py:14-71; args of continuous_mountain_car.py:105-121).
 * action float32 [E,1,1]. */
int wdb_continuous_mountain_car_step(void *stream, int n_envs, float *state,
                                     const float *action, int *done, float *reward,
                                     float *obs, float min_action, float max_action,
                                     float min_position, float max_position, float max_speed,
                                     float goal_position, float goal_velocity, float power,
                                     int *env_timestep, int episode_length);

/* Replaces NumbaClassicControlPendulumEnvStep (pendulum/pendulum_step_numba.py:30-72; args
 * of pendulum.py:92-100).  state k = 2 (theta, theta_dot), obs k = 3, action float32. */
int wdb_pendulum_step(void *stream, int n_envs, float *state, const float *action, int *done,
                      float *reward, float *obs, int *env_timestep, int episode_length);

/* Replaces NumbaClassicControlAcrobotEnvStep (acrobot/acrobot_step_numba.py:24-168; args of
 * acrobot.py:91-99).  state k = 4 (16-byte aligned), obs k = 6, action int32 in {0,1,2}. */
int wdb_acrobot_step(void *stream, int n_envs, float *state, const int *action, int *done,
                     float *reward, float *obs, int *env_timestep, int episode_length);

/* ------------------------------------------ whole rollout, single-agent envs ---- */
/* ONE launch = n_steps rollout timesteps of a single-agent classic-control env, one thread
 * per env replica: FullyConnected forward (fp32, weights in shared memory) -> action sample
 * -> step -> bookkeeping -> done-masked reset -> push to the batch slots.  Replaces the body
 * of TrainerBase._generate_rollout_batch (trainer_base.py:383-428) for
 * ClassicControl{CartPole,MountainCar,Acrobot}Env, and the DDPG rollout of
 * ClassicControl{ContinuousMountainCar,Pendulum}Env (trainer_ddpg.py): per timestep the
 * reference issues the model forward, sample_actions / sample_ou_process, Numba...EnvStep,
 * ~20 bookkeeping torch ops and one reset kernel per registered array.
 * Discrete kinds: softmax head, categorical sample, int32 actions.  Continuous kinds: a head
 * of width 1, mean = action_scale * tanh(z) + action_bias, OU noise exactly as
 * wdb_sample_ou_process (stream = env), float32 actions.  The step physics and the OU update
 * are the same compiled functions the stand-alone kernels call. */
enum {
  WDB_SA_CARTPOLE = 0, WDB_SA_MOUNTAIN_CAR = 1, WDB_SA_ACROBOT = 2,
  WDB_SA_CONTINUOUS_MOUNTAIN_CAR = 3,  /* state 2, obs 2, done at episode end or goal */
  WDB_SA_PENDULUM = 4                  /* state 2, obs 3, done at episode end */
};

typedef struct wdb_sa_rollout {
  int env_kind, n_envs, n_steps, episode_length, state_dim, use_argmax;
  float env_params[12];              /* the scalar arguments of the env's step function, in
                                      * the order of wdb_cartpole_step / wdb_mountain_car_step /
                                      * wdb_continuous_mountain_car_step (Pendulum: none) */
  float *state;                      /* [E, state_dim] */
  float *observations;               /* [E, F] current observation (read and updated) */
  int *done, *env_timestep;          /* [E] */
  float *rewards;                    /* [E] */
  void *sampled_actions;             /* [E]: int32 (discrete kinds) or float32 (continuous) */
  int n_hidden;                      /* hidden Linear + ReLU layers (0..3), then the head */
  int dims[5];                       /* F, H1, ..., A: F = the kind's observation width, A =
                                      * its action count (CartPole 2, MountainCar 3, Acrobot
                                      * 3; continuous kinds 1); hidden widths 1..64 */
  const float *w[4], *b[4];          /* nn.Linear weights [out, in] and biases, fp32 */
  void *rng_state;
  const float *uniforms;             /* test hook [n_steps, E]; NULL = device RNG */
  float *obs_batch;                  /* [n_steps, E, F] or NULL */
  void *actions_batch;               /* [n_steps, E] or NULL; element type of sampled_actions */
  float *rewards_batch;              /* [n_steps, E] or NULL */
  int *done_batch;                   /* [n_steps, E] or NULL */
  float *probs_batch;                /* [n_steps, E, A] or NULL (tests); continuous: the mean */
  float *reward_running_sum;         /* [E] or NULL */
  int *step_running_sum;             /* [E] or NULL */
  float *episodic_reward_sum;        /* scalar or NULL */
  unsigned long long *episodic_step_sum, *num_completed;   /* scalars or NULL */
  const wdb_reset_desc *reset_table; /* device table of the arrays to restore when done */
  int n_reset_arrays;
  void *pool_rng;                    /* RNG state of the reset pools, or NULL */
  int reset_done_envs;
  /* continuous kinds only (ignored otherwise) */
  float ou_damping, ou_stddev, ou_scale;  /* as wdb_sample_ou_process; scale < 1e-8: no noise */
  float *ou_state;                   /* [E] OU state; required unless scale < 1e-8 */
  float action_scale, action_bias;   /* the actor's output_w / output_b */
  const float *normals;              /* test hook [n_steps, E]; NULL = device RNG */
  /* continuous kinds, Gaussian head (gaussian_head = 1): the head's raw output is the mean of a
   * diagonal Gaussian and the action is sampled as wdb_sample_gaussian (stream = env; no tanh,
   * no scale / bias, no OU state; use_argmax: action = mean).  0: the tanh + OU head above.
   * Continuous kinds, squashed Gaussian head (gaussian_head = 2; SAC's actor): the head is 2
   * wide, [mu, raw log-std], and the action is sampled as wdb_sample_squashed_gaussian
   * (stream = env): action_scale * tanh(mu + exp(clamp(log-std, log_std[0], log_std[1])) n) +
   * action_bias (use_argmax: u = mu).  No OU state. */
  const float *log_std;              /* required with gaussian_head: [1] the log-std (1), or
                                      * [2] the log-std's clamp bounds min <= max (2) */
  int gaussian_head;                 /* 0: tanh + OU, 1: Gaussian, 2: squashed Gaussian,
                                      * 3: Gaussian on normalized observations; discrete
                                      * kinds: 3 = Q head, 4 = categorical Q head, 5 = noisy
                                      * Q head, 6 = softmax on normalized observations, else
                                      * softmax */
  /* Discrete kinds, Q head (gaussian_head = 3; DQN's FullyConnectedQ): the head's raw outputs
   * are Q values, written to probs_batch when given, and the action is sampled as
   * wdb_sample_epsilon_greedy (stream = env, one draw per step) with epsilon = log_std[0], a
   * device float in [0, 1] (use_argmax: epsilon = 0).  Needs log_std and rng_state; `uniforms`
   * must be NULL.  (The struct keeps its layout.)
   * Discrete kinds, categorical Q head (gaussian_head = 4; C51's FullyConnectedCategoricalQ):
   * the head is A blocks of N atom logits, dims[n_hidden + 1] = A * N with A the kind's action
   * count.  Each block is reduced to Q[a] = sum_j z_j softmax_j over the env's 8 lanes (lane k:
   * j = k, k + 8, ... in order, then an xor butterfly; e_j = expf(y_j - max y), Q = (sum z_j
   * e_j) / (sum e_j)); Q is written to probs_batch when given and sampled as the Q head is.
   * log_std = [epsilon, z_0, ..., z_{N-1}] on the device.
   * Discrete kinds, noisy Q head (gaussian_head = 5; FullyConnectedQ with a noisy output layer):
   * w / b of the head are mu_W, mu_b.  log_std = [epsilon, key words, sigma_W [A][H], sigma_b
   * [A]] on the device, the four key words (raw 32-bit: seed low, seed high, step low, step
   * high) giving the noise of wdb_noisy_* in the acting domain, layer 0, counter row = env, step
   * = the given step + t at timestep t.  Output j = fmaf(f(eps_out)_j, s_j, m_j): m_j the Q head's
   * output (bias, then fmaf over the inputs in order), s_j = sigma_b_j then fmaf(sigma_W[j][i],
   * f(eps_in)_i * h_i, .) over i in order; use_argmax: m_j alone (the mean network) and epsilon
   * 0.  Then sampled as the Q head is.
   * Normalized observations (gaussian_head = 6 on a discrete kind: the softmax head; 3 on a
   * continuous kind: the Gaussian head): each observation element x enters the first layer as
   * clamp((x - shift_i) * scale_i, -clip, clip) (a rounded subtract, then a rounded multiply,
   * then the clamp: wdb_obs_normalize's arithmetic); obs_batch keeps the raw x.  log_std =
   * [shift F | scale F | clip] on the device, after the log-std for the Gaussian head. */
} wdb_sa_rollout;

int wdb_single_agent_rollout_supported(int n_hidden, const int *dims);
/* 1 if a categorical Q head of dims[n_hidden + 1] = A * N outputs runs in one launch: the
 * hidden widths and F as wdb_single_agent_rollout_supported takes them, 2 <= N <= 64, N
 * dividing the head, and the same cap on the network's floats. */
int wdb_single_agent_rollout_categorical_supported(int n_hidden, const int *dims, int n_atoms);
/* 1 if a noisy Q head runs in one launch: the shapes of wdb_single_agent_rollout_supported, A
 * <= 8, and the network's floats plus the head's A * H + A sigma floats within the same cap. */
int wdb_single_agent_rollout_noisy_supported(int n_hidden, const int *dims);
int wdb_single_agent_rollout(void *stream, const wdb_sa_rollout *rollout);

/* -------------------------------------------------- rollout of ANY env: data movement ---- */
/* [E, N, W] array of 4-byte elements <-> one dense [E, Np, W] block per policy, every policy
 * in one launch.  scatter = 0: rows[e, j, :] = full[e, agent_ids[j], :] (the per-policy
 * observation push of warp_drive/training/trainer_base.py:437-464); scatter = 1: the reverse
 * (the per-policy probabilities into the [E, N, A] array the sampler reads, :466-512).
 * agent_ids == NULL: the policy covers agents 0..Np-1 in order. */
typedef struct wdb_gather_policy {
  int n_agents;                      /* Np */
  const int *agent_ids;              /* device [Np] or NULL */
  void *rows;                        /* [E, Np, W] */
} wdb_gather_policy;
typedef struct wdb_gather {
  int n_envs, n_agents, width, n_policies, scatter;
  void *full;                        /* [E, N, W] */
  wdb_gather_policy policy[4];
} wdb_gather;
int wdb_gather_policy_rows(void *stream, const wdb_gather *gather);

/* Dict observations: several [E, N, width] source arrays (one per key of the Dict, int32 or
 * float32) into up to two dense float32 destinations per policy, every field of every policy
 * in one launch.  Field f of agent agent_ids[j] lands, converted to float32, at columns
 * [col, col + width) of row (e, j) of destination `dst` of the policy: destination 0 is the
 * processed observation [E, Np, dst_width[0]] (the non-mask keys concatenated), destination 1
 * the action-mask rows [E, Np, dst_width[1]].  A NULL destination is skipped.
 * Heterogeneous agents (a zero-initialised extension keeps the behaviour above):
 *   policy_mask  bit p set: the field feeds policy p only; 0 = every policy;
 *   own_rows     1: src holds only its policy's agents, in slot order (Ns = Np, agent_ids
 *                unused; policy_mask must name exactly one policy); 0: every agent (Ns = N);
 *   agents_last  1: src is [E, *F, Ns] with width = prod(F): column c of agent a of env e is
 *                src[(e * width + c) * Ns + a] (C order over F, numpy.moveaxis(x, 0, -1) of
 *                [Ns, *F]); moved through a shared-memory tile so that reads and writes are
 *                both coalesced;
 *   policy[p].dst_width[d] > 0 overrides dst_width[d] for that policy. */
#define WDB_GATHER_MAX_FIELDS 16
typedef struct wdb_gather_field {
  const void *src;                   /* [E, Ns, width] or [E, width, Ns] */
  int width, is_int32, dst, col;
  int policy_mask, own_rows, agents_last;
} wdb_gather_field;
typedef struct wdb_gather_fields_policy {
  int n_agents;                      /* Np */
  const int *agent_ids;              /* device [Np] or NULL (agents 0..Np-1) */
  float *rows[2];                    /* [E, Np, dst_width[d]] or NULL */
  int dst_width[2];                  /* 0: the descriptor's dst_width[d] */
} wdb_gather_fields_policy;
typedef struct wdb_gather_fields {
  int n_envs, n_agents, n_policies, n_fields;
  int dst_width[2];
  wdb_gather_field field[WDB_GATHER_MAX_FIELDS];
  wdb_gather_fields_policy policy[4];
} wdb_gather_fields;
int wdb_gather_policy_fields(void *stream, const wdb_gather_fields *gather);

/* Per-timestep bookkeeping of the rollout (trainer_base.py:514-601, which uses
 * done_flags.nonzero() and len() on the host): done -> done_batch (raw flag); per policy the
 * agents' rewards -> rewards_batch, sampled actions -> actions_batch, reward_running_sum += r,
 * and for done envs episodic_reward_sum += the running sums, which are then cleared;
 * step_running_sum += 1, for done envs episodic_step_sum += it, cleared, num_completed += 1.
 * Any pointer may be NULL (that piece is skipped); ONE launch, no host synchronisation.
 * A policy with its own step arrays (separate placeholders) sets policy[p].rewards [E, Np]
 * and / or policy[p].actions [E, Np, policy[p].n_heads]; those are read in slot order instead
 * of the shared rewards / actions through agent_ids.  The shared rewards may be NULL when
 * every policy has its own. */
typedef struct wdb_bookkeep_policy {
  int n_agents;
  const int *agent_ids;              /* device [Np] or NULL (agents 0..Np-1) */
  float *rewards_batch;              /* [E, Np] slot t */
  int *actions_batch;                /* [E, Np, n_heads] slot t */
  float *reward_running_sum;         /* [E, Np] */
  float *episodic_reward_sum;        /* scalar */
  const float *rewards;              /* [E, Np] or NULL (the shared rewards) */
  const int *actions;                /* [E, Np, n_heads] or NULL (the shared actions) */
  int n_heads;                       /* heads of `actions` (ignored when it is NULL) */
} wdb_bookkeep_policy;
typedef struct wdb_bookkeep {
  int n_envs, n_agents, n_policies, n_heads;
  const int *done;                   /* [E] */
  const float *rewards;              /* [E, N] or NULL */
  const int *actions;                /* [E, N, n_heads] or NULL */
  int *done_batch;                   /* [E] slot t */
  int *step_running_sum;             /* [E] */
  unsigned long long *episodic_step_sum, *num_completed_episodes;
  wdb_bookkeep_policy policy[4];
} wdb_bookkeep;
int wdb_rollout_bookkeep(void *stream, const wdb_bookkeep *bookkeep);

/* ------------------------------------------------------------- policy forward ---- */
/* Fused policy/value MLP forward on the tensor cores (wgmma), replacing the
 * rollout-time FullyConnected.forward (warp_drive/training/models/fully_connected.py:51-89):
 *   obs [rows, F] -> Linear(F,H)+ReLU -> Linear(H,H)+ReLU -> softmax(Linear(H,A0)),
 *   softmax(Linear(H,A1)), Linear(H,1).
 * Weights are nn.Linear tensors ([out, in] fp32); wdb_mlp_pack_weights converts them to bf16
 * tiles inside a caller-owned blob of wdb_mlp_blob_bytes() bytes (re-pack after every
 * optimizer step).  H must be a multiple of 32 <= 256, A0 + A1 + 1 <= 64, F <= 256;
 * wdb_mlp_blob_bytes returns -1 for unsupported shapes. */
long long wdb_mlp_blob_bytes(int F, int H, int A0, int A1);
int wdb_mlp_pack_weights(void *stream, void *blob, const float *w1, const float *b1,
                         const float *w2, const float *b2, const float *wh0, const float *bh0,
                         const float *wh1, const float *bh1, const float *wv, const float *bv,
                         int F, int H, int A0, int A1);
int wdb_mlp_policy_forward(void *stream, const void *blob, int F, int H, int A0, int A1,
                           const float *obs, long long rows, float *probs0, float *probs1,
                           float *values /* may be NULL */);
/* The same forward with an action mask [rows, A0 + A1] f32 (1 = valid, 0 = invalid; head 0's
 * columns first): (1 - m) * -1e20 is added to each action logit in fp32 before the softmax,
 * as FullyConnected's apply_logit_mask does.  Masked probabilities come out exactly 0, and a
 * head with every action masked comes out uniform. */
int wdb_mlp_policy_forward_masked(void *stream, const void *blob, int F, int H, int A0, int A1,
                                  const float *obs, long long rows, const float *mask,
                                  float *probs0, float *probs1, float *values /* may be NULL */);
/* The same forward, which also samples both heads of every row as the fused TagContinuous
 * step samples them (wdb_sample_actions): row r = env * Np + slot is agent
 * gi = env * N + agent_of_slot[slot]; its uniforms are draws x (head 0) and y (head 1) of
 * Philox stream gi at that stream's offset, which advances by one (or uniforms[2 gi + head]
 * when `uniforms` is set; the offsets are then left alone).  actions[r] = (head 0, head 1)
 * is the index the reference's CDF search picks from the stored probabilities.  Only the
 * config-2 shape samples (F in [65, 80], H = 256, two heads with A0 + A1 + 1 in [33, 48]):
 * wdb_mlp_forward_samples says whether a shape does.  input_is_tiles: `input` is the bf16
 * tile copy of wdb_mlp_policy_forward_tiles instead of fp32 obs [rows, F]. */
typedef struct wdb_mlp_sampling {
  int *actions;                      /* [rows, 2] (8-byte aligned) */
  void *rng_state;                   /* wdb_rng_init state of E * N streams; may be NULL with uniforms */
  const float *uniforms;             /* [E, N, 2] or NULL */
  const int *agent_of_slot;          /* [Np] */
  int n_agents;                      /* N */
  int n_policy_agents;               /* Np; rows must be a multiple of it */
  long long row_offset;              /* the launch's rows are rows [row_offset, + rows) of the
                                      * policy (a multiple of Np): row r samples agent
                                      * (row_offset + r) / Np * N + agent_of_slot[...]; actions
                                      * and every other row array start at the launch's row 0 */
} wdb_mlp_sampling;
int wdb_mlp_forward_samples(int F, int H, int A0, int A1);
int wdb_mlp_policy_forward_sampled(void *stream, const void *blob, int F, int H, int A0, int A1,
                                   const void *input, int input_is_tiles, long long rows,
                                   float *probs0, float *probs1, float *values /* may be NULL */,
                                   const wdb_mlp_sampling *sampling);
/* Two policies in ONE launch (the rollout of a two-policy env: tag_continuous runners and
 * taggers): CTAs [0, grid - ctas_b) run policy 0, the last ctas_b CTAs policy 1, each
 * persistent over its own 128-row tiles.  ctas_b = 0 picks the split from the row counts.
 * flags: WDB_MLP_WEIGHTS_STABLE = neither blob was written by the kernel launched just before
 * this one on `stream` (true for every rollout step but the first after a weight re-pack): with
 * the "pdl" option on, the launch is a programmatic dependent launch and the weight load then
 * overlaps the tail of that previous kernel. */
#define WDB_MLP_WEIGHTS_STABLE 1
typedef struct wdb_mlp_pair {
  const void *blob[2];
  int F[2], H[2], A0[2], A1[2];
  const float *obs[2];
  long long rows[2];
  float *probs0[2], *probs1[2], *values[2];   /* values may be NULL */
  int ctas_b;
  int flags;
} wdb_mlp_pair;
int wdb_mlp_policy_forward_pair(void *stream, const wdb_mlp_pair *pair);

/* The same forward fed from the bf16 copy of the observations in A-operand layout: 128-row
 * tiles, each one contiguous block (canonical K-major layout, K padded to a multiple of 16
 * with zeros) that the kernel fetches with one TMA bulk copy.  wdb_mlp_pack_obs builds it
 * from fp32 obs [rows, F]; the fused tag_continuous step writes it directly
 * (wdb_tc_policy_io.obs_next_tiles).  No reference counterpart: the reference always runs
 * the torch forward on the fp32 batch slice (trainer_base.py:437-464). */
long long wdb_mlp_obs_tiles_bytes(int F, long long rows);
int wdb_mlp_pack_obs(void *stream, const float *obs, long long rows, int F, void *tiles);
int wdb_mlp_policy_forward_tiles(void *stream, const void *blob, int F, int H, int A0, int A1,
                                 const void *obs_tiles, long long rows, float *probs0,
                                 float *probs1, float *values /* may be NULL */);

/* ------------------------------------------------------------------ update ---- */
/* Bootstrapped discounted returns of the A2C/PPO update, backwards in time with done
 * masking (warp_drive/training/algorithms/policygradient/a2c.py:80-93):
 *   returns[T-1] = done ? r : V ;  returns[t] = r[t] + (done[t] ? 0 : gamma*returns[t+1]).
 * rewards/values/returns [T, E, Np] f32, done [T, E] i32. */
int wdb_discounted_returns(void *stream, const float *rewards, const int *done,
                           const float *values, float *returns, int T, int n_envs,
                           int n_agents, float gamma);

/* Elementwise pieces of the MLP's TRAINING forward / backward (warp_drive/training/models/
 * fully_connected.py:51-89 under autograd); the GEMMs between them stay on cuBLAS.
 * wdb_heads_softmax: logits [rows, pitch >= A0 + A1 + 1] (the pitch is padded to a multiple of
 * 4 floats so that cuBLAS can use its 16-byte-aligned tensor-core kernels; wdb_heads_softmax_backward
 * zero-fills the padding columns) of the two action heads and the value head
 * (one GEMM) -> softmax per head into probs0 [rows, A0], probs1 [rows, A1] (A1 may be 0) and
 * the value column into values [rows].  wdb_heads_softmax_backward: the gradient with respect
 * to those logits from the gradients of probs / values (NULL = no gradient).
 * wdb_relu_backward_bias: grad_hidden[r, c] = hidden[r, c] > 0 ? grad_hidden[r, c] : 0 in
 * place, and per CTA the column sums of the result into partial_bias_grads
 * [ceil(rows / wdb_relu_backward_bias_rows(rows)), width] (the bias gradient = their sum;
 * no atomics: deterministic). */
int wdb_heads_softmax(void *stream, const float *logits, long long rows, int A0, int A1,
                      int pitch, float *probs0, float *probs1, float *values);
/* wdb_heads_softmax with an action mask [rows, mask_pitch] f32, A0 + A1 <= mask_pitch <= pitch
 * (1 = valid): (1 - m) * -1e20 is added to each action logit before its head's softmax.  The
 * backward needs no mask: a probability of 0 gives a logit gradient of 0.  Takes the shapes
 * wdb_heads_softmax_supported accepts. */
int wdb_heads_softmax_masked(void *stream, const float *logits, long long rows, int A0, int A1,
                             int pitch, const float *mask, int mask_pitch, float *probs0,
                             float *probs1, float *values);
int wdb_heads_softmax_backward(void *stream, const float *probs0, const float *probs1,
                               const float *grad_probs0, const float *grad_probs1,
                               const float *grad_values, long long rows, int A0, int A1,
                               int pitch, float *grad_logits);
/* 1 if BOTH wdb_heads_softmax and wdb_heads_softmax_backward take heads of A0 / A1 actions at
 * this logits pitch (the backward stages two row tiles: it takes pitches below 200, the
 * forward below 400), else 0.  The launches refuse exactly the shapes this refuses. */
int wdb_heads_softmax_supported(int A0, int A1, int pitch);
int wdb_pad_rows(void *stream, const float *src, long long rows, int width, int pitch,
                 float *dst /* [rows, pitch], columns >= width zero-filled */);
int wdb_relu_backward_bias_rows(long long rows);
int wdb_relu_backward_bias(void *stream, float *grad_hidden, const float *hidden,
                           long long rows, int width, float *partial_bias_grads);

/* Fused A2C / PPO loss (a2c.py:80-130, ppo.py:82-141): ONE backward-in-time scan per (env,
 * agent) computes the bootstrapped returns, advantages, Categorical log-prob and entropy of
 * every head, the loss sums and the gradients of
 *     loss = mean(-logp * adv) + vf_coeff * mean((V - R)^2) - entropy_coeff * sum_k mean(H_k)
 * with respect to the probabilities and the values (PPO's clipped surrogate has the same
 * gradient at ratio == 1, the reference's single-epoch case, ppo.py:127-136; several epochs
 * over minibatches go through wdb_gae and wdb_ppo_loss_and_grads).
 * sums (double[4], zeroed by the caller): sum(-logp*adv), sum((V-R)^2), sum_k sum(H_k), sum(adv). */
typedef struct wdb_pg_loss {
  int T, n_envs, n_agents, n_heads;
  int n_actions[4];
  const float *probs[4];             /* [T, E, Np, A_k] */
  const float *values;               /* [T, E, Np] */
  const int *actions;                /* [T, E, Np, n_heads] */
  const float *rewards;              /* [T, E, Np] */
  const int *done;                   /* [T, E] (non-zero = done) */
  float gamma, vf_coeff, entropy_coeff;
  float *grad_probs[4];              /* out, same shapes as probs (or NULL) */
  float *grad_values;                /* out (or NULL) */
  float *returns;                    /* out [T, E, Np] (or NULL) */
  double *sums;                      /* out [4], accumulated atomically */
} wdb_pg_loss;
int wdb_pg_loss_and_grads(void *stream, const wdb_pg_loss *loss);
/* 1 if wdb_pg_loss_and_grads takes n_heads heads of n_actions[k] actions (1..4 heads, each of
 * 1..399 actions: one 32-row tile of the widest head per warp), else 0.  No CUDA call. */
int wdb_pg_loss_supported(int n_heads, const int *n_actions);

/* The same fused A2C / PPO loss for a diagonal Gaussian policy with a state-independent log-std
 * (FullyConnectedGaussian; the reference has no counterpart).  Returns, advantages and done
 * masking as wdb_pg_loss_and_grads; per row, with z_k = (a_k - mu_k) * exp(-ls_k):
 *   logp = sum_k -z_k^2 / 2 - ls_k - log(2 pi) / 2,   H = sum_k ls_k + (1 + log(2 pi)) / 2,
 *   loss = mean(-logp * adv) + vf_coeff * mean((V - R)^2) - entropy_coeff * mean(H)
 * (PPO at ratio == 1 has the same gradient).  Outputs: the gradient with respect to the mean
 * (per row), the values (per row) and log_std (reduced over every row: per-CTA float64
 * partials summed in a fixed order by a second kernel, so it is bit-identical on relaunch),
 * the float64 sums of wdb_pg_loss_and_grads, and optionally the returns.  Two launches. */
#define WDB_PG_GAUSSIAN_MAX_DIM 8
#define WDB_PG_GAUSSIAN_ROWS_PER_CTA 128
typedef struct wdb_pg_gaussian_loss {
  int T, n_envs, n_agents, action_dim;   /* action_dim A: 1..WDB_PG_GAUSSIAN_MAX_DIM */
  const float *mean;                 /* [T, E, Np, A] */
  const float *log_std;              /* [A] */
  const float *values;               /* [T, E, Np] */
  const float *actions;              /* [T, E, Np, A] f32 */
  const float *rewards;              /* [T, E, Np] */
  const int *done;                   /* [T, E] (non-zero = done) */
  float gamma, vf_coeff, entropy_coeff;
  float *grad_mean;                  /* out [T, E, Np, A] (or NULL) */
  float *grad_log_std;               /* out [A] (or NULL) */
  float *grad_values;                /* out [T, E, Np] (or NULL) */
  float *returns;                    /* out [T, E, Np] (or NULL) */
  double *sums;                      /* out [4] as wdb_pg_loss, accumulated atomically */
  double *partials;                  /* workspace [ceil(E * Np / ROWS_PER_CTA), A] doubles;
                                      * required with grad_log_std */
} wdb_pg_gaussian_loss;
int wdb_pg_gaussian_loss_and_grads(void *stream, const wdb_pg_gaussian_loss *loss);
/* 1 if wdb_pg_gaussian_loss_and_grads takes this action dimension (1..WDB_PG_GAUSSIAN_MAX_DIM:
 * a row's dimensions are held in registers), else 0.  No CUDA call. */
int wdb_pg_gaussian_loss_supported(int action_dim);

/* Multi-epoch PPO over shuffled minibatches (no reference counterpart: the reference's PPO
 * takes one step per batch at ratio == 1).
 *
 * wdb_gae: advantages and value targets of GAE(lambda), one backward-in-time scan per (env,
 * agent), with d = done[t, e] > 0 and the bootstrapping of wdb_discounted_returns:
 *   t = T-1:  A = d ? r - V : 0
 *   t < T-1:  delta = r + (d ? 0 : gamma * V[t+1]) - V ;  A = delta + (d ? 0 : gamma*lambda*A[t+1])
 *   value_target = A + V
 * (lambda = 1: value_target is the discounted return; lambda = 0: one-step TD). */
typedef struct wdb_gae_args {
  int T, n_envs, n_agents;
  const float *rewards;              /* [T, E, Np] */
  const float *values;               /* [T, E, Np] */
  const int *done;                   /* [T, E] (> 0 = done) */
  float gamma, gae_lambda;
  float *advantages;                 /* out [T, E, Np] */
  float *value_targets;              /* out [T, E, Np] */
} wdb_gae_args;
int wdb_gae(void *stream, const wdb_gae_args *gae);

/* The loss of one minibatch of B rows of the flat [R = T * E * Np] batch and its gradients with
 * respect to the model outputs.  Row b of the minibatch is flat row rows[b] (rows == NULL: row
 * b); the model outputs (probs / mean, values) are in minibatch order, everything else is read
 * through rows.  With l = the row's log-prob (Categorical over every head, as
 * wdb_pg_loss_and_grads, or the diagonal Normal of wdb_pg_gaussian_loss_and_grads),
 * rho = exp(l - old_log_prob), A = advantages and eps = clip_param:
 *   policy = ppo ? -(1/B) sum min(rho * A, clamp(rho, 1 - eps, 1 + eps) * A)
 *                : -(1/B) sum l * A
 *   loss   = policy + vf_coeff * (1/B) sum (V - value_target)^2 - entropy_coeff * (1/B) sum H
 * The gradients are torch autograd's for that expression: torch.minimum gives half to each side
 * of a tie, clamp passes the gradient on the closed interval [1 - eps, 1 + eps].
 * sums (double[5], zeroed by the caller): sum of the policy terms, sum (V - value_target)^2,
 * sum H, sum (old_log_prob - l) (approximate KL), count of |rho - 1| > eps.
 * log_prob (optional out [B]): l in minibatch order.  old_log_prob == NULL is the log-prob
 * pre-pass: only log_prob is written (required), no gradient output may be given, and values,
 * advantages, value_targets and sums are not read. */
typedef struct wdb_ppo_loss {
  int B, n_heads;
  int n_actions[4];
  const float *probs[4];             /* [B, A_k] */
  const float *values;               /* [B] */
  const int *rows;                   /* [B] into [R], or NULL */
  const int *actions;                /* [R, n_heads] */
  const float *advantages;           /* [R] */
  const float *value_targets;        /* [R] */
  const float *old_log_prob;         /* [R], or NULL: the pre-pass */
  int ppo;                           /* 0: the A2C policy term */
  float clip_param, vf_coeff, entropy_coeff;
  float *grad_probs[4];              /* out [B, A_k] (or NULL) */
  float *grad_values;                /* out [B] (or NULL) */
  float *log_prob;                   /* out [B] (or NULL) */
  double *sums;                      /* out [5], accumulated atomically */
} wdb_ppo_loss;
int wdb_ppo_loss_and_grads(void *stream, const wdb_ppo_loss *loss);
/* 1 if wdb_ppo_loss_and_grads takes these heads (those of wdb_pg_loss_supported), else 0.
 * No CUDA call. */
int wdb_ppo_loss_supported(int n_heads, const int *n_actions);

/* The same for a diagonal Gaussian policy.  The log_std gradient,
 *   -(1/B) sum_b w_b (z_bk^2 - 1) - entropy_coeff  with w_b = -B * d policy / d l_b,
 * is summed from per-CTA float64 partials in a fixed order by a second launch, so it is
 * bit-identical on relaunch. */
typedef struct wdb_ppo_gaussian_loss {
  int B, action_dim;                 /* action_dim A: 1..WDB_PG_GAUSSIAN_MAX_DIM */
  const float *mean;                 /* [B, A] */
  const float *log_std;              /* [A] */
  const float *values;               /* [B] */
  const int *rows;                   /* [B] into [R], or NULL */
  const float *actions;              /* [R, A] */
  const float *advantages;           /* [R] */
  const float *value_targets;        /* [R] */
  const float *old_log_prob;         /* [R], or NULL: the pre-pass */
  int ppo;
  float clip_param, vf_coeff, entropy_coeff;
  float *grad_mean;                  /* out [B, A] (or NULL) */
  float *grad_log_std;               /* out [A] (or NULL) */
  float *grad_values;                /* out [B] (or NULL) */
  float *log_prob;                   /* out [B] (or NULL) */
  double *sums;                      /* out [5] as wdb_ppo_loss */
  double *partials;                  /* workspace [ceil(B / ROWS_PER_CTA), A] doubles;
                                      * required with grad_log_std */
} wdb_ppo_gaussian_loss;
int wdb_ppo_gaussian_loss_and_grads(void *stream, const wdb_ppo_gaussian_loss *loss);
/* 1 if wdb_ppo_gaussian_loss_and_grads takes this action dimension, else 0.  No CUDA call. */
int wdb_ppo_gaussian_loss_supported(int action_dim);

/* Gradient-norm clipping + Adam over one flat float32 arena (torch.optim.Adam semantics, no
 * weight decay; torch.nn.utils.clip_grad_norm_ semantics for the clip factor, which the Adam
 * kernel reads from device memory: no host synchronisation).  Replaces the per-tensor
 * optimizer loop of trainer_a2c.py:300-339. */
int wdb_grad_sumsq(void *stream, const float *grads, long long n, double *out /* += */);
int wdb_adam_step(void *stream, float *params, float *grads, float *exp_avg, float *exp_avg_sq,
                  long long n, float lr, float beta1, float beta2, float eps, int step,
                  float max_grad_norm /* <= 0: no clipping */, const double *grad_sumsq);

/* Every gradient of one DDPG update of one policy (trainer_ddpg.py:380-420,
 * algorithms/ddpg.py:62-120 of the reference) read in place from the replay ring: logical slot
 * k is physical slot (cursor + k) mod capacity, k = 0 the oldest.  With valid = capacity -
 * n_step + 1 and M = valid * E * Np loss rows:
 *   critic_loss = mean over the loss rows of (Q(obs, actions) - R)^2,
 *   actor_loss  = -mean of J = Q(obs, actor(obs)),
 *   R = the n-step return bootstrapped with target_critic(obs', target_actor(obs')) at slot
 *       i + n_step (the last window: slot capacity - 1, undiscounted, ddpg.py:68-73),
 * the actor gradient = d actor_loss, the critic gradient = d critic_loss + d actor_loss (the
 * reference's actor_loss.backward() also reaches the critic).  Networks: hidden Linear + ReLU
 * layers, then the head (the critic's input is obs ++ action; the actor's output is
 * action_scale * tanh(z) + action_bias).  Float32 FMA; the per-CTA partial gradients are
 * summed in a fixed order by a second kernel that writes them to gw / gb: no float atomics,
 * bit-reproducible.  Two launches. */
typedef struct wdb_ddpg_net {
  int n_hidden;                      /* 0..3 */
  int widths[3];                     /* hidden widths (1..64) */
  const float *w[4], *b[4];          /* nn.Linear weights [out, in] and biases, hidden then head */
  float *gw[4], *gb[4];              /* gradients, same shapes (actor / critic; NULL for targets) */
} wdb_ddpg_net;
typedef struct wdb_ddpg_update_args {
  int n_envs, n_agents, obs_dim, action_dim;   /* E, Np, F, A */
  int capacity, cursor, n_step;      /* ring slots C, oldest slot, n-step horizon (1..C) */
  float gamma, action_scale, action_bias;
  const float *obs;                  /* [C, E, Np, F] */
  const float *actions;              /* [C, E, Np, A] */
  const float *rewards;              /* [C, E, Np] */
  const int *done;                   /* [C, E] */
  wdb_ddpg_net actor, critic, target_actor, target_critic;   /* targets: the online shapes */
  float *values, *j_values, *returns;  /* out [valid, E * Np] in logical slot order, or NULL */
  double *sums;                      /* out [2]: sum (Q - R)^2, sum J over the loss rows */
  void *workspace;                   /* wdb_ddpg_update_workspace_bytes() bytes */
} wdb_ddpg_update_args;
/* 1 if the shapes are supported: 0..3 hidden layers of width 1..64 per network, F + A <= 64,
 * targets shaped as the online networks, E, Np >= 1, 1 <= n_step <= capacity, capacity >= 2
 * (the last window's bootstrap value is the target critic at slot capacity - 1), cursor in
 * [0, capacity), and all four networks' weights, the gradient accumulators and a row tile fit
 * one CTA's shared memory (227 KB).  No CUDA call. */
int wdb_ddpg_update_supported(const wdb_ddpg_update_args *update);
long long wdb_ddpg_update_workspace_bytes(const wdb_ddpg_update_args *update);  /* -1: unsupported */
/* cudaErrorInvalidValue without launching if unsupported or a required pointer is NULL. */
int wdb_ddpg_update(void *stream, const wdb_ddpg_update_args *update);

/* One TD3 update of one policy (Fujimoto et al. 2018) over the same ring and the same M loss
 * rows as wdb_ddpg_update, as two passes of two launches each (a tile kernel and the
 * fixed-order reduction: bit-reproducible).
 * Critic pass (wdb_td3_critic_update): per loss row g (window i, agent row n) and action dim c,
 *   a'[c] = clamp(pi'[c] + clamp(sigma * scale * noise[g][c], -clip * scale, clip * scale),
 *                 bias - scale, bias + scale),   pi' = target_actor(obs') as in DDPG,
 *   R = the n-step return of DDPG bootstrapped with min(target_critic(obs', a'),
 *       target_critic2(obs', a')) at DDPG's bootstrap slot,
 *   gradients of mse(Q1(obs, actions), R) + mse(Q2(obs, actions), R) into critic.gw / gb and
 *   critic2.gw / gb (nothing else reaches them).
 * Actor pass (wdb_td3_actor_update): the gradient of -mean Q1(obs, actor(obs)) into
 *   actor.gw / gb (the critic's weights carry it to the action inputs; no critic gradient).
 * The critic pass reads critic, critic2, both target critics and target_actor; the actor pass
 * reads actor and critic. */
typedef struct wdb_td3_update_args {
  int n_envs, n_agents, obs_dim, action_dim;   /* E, Np, F, A */
  int capacity, cursor, n_step;      /* as wdb_ddpg_update_args */
  float gamma, action_scale, action_bias;
  float target_noise, target_noise_clip;       /* sigma, clip >= 0: units of action_scale */
  const float *obs;                  /* [C, E, Np, F] */
  const float *actions;              /* [C, E, Np, A] */
  const float *rewards;              /* [C, E, Np] */
  const int *done;                   /* [C, E] */
  const float *noise;                /* [valid, E * Np, A] standard normal, logical window order */
  wdb_ddpg_net actor, critic, critic2;          /* gradients: actor (actor pass), critics */
  wdb_ddpg_net target_actor, target_critic, target_critic2;   /* the online shapes */
  float *q1_values, *q2_values, *returns;       /* critic pass out [valid, E * Np], or NULL */
  float *j_values;                   /* actor pass out [valid, E * Np], or NULL */
  double *sums;                      /* out [4]: sum (Q1 - R)^2, sum (Q2 - R)^2 (critic pass),
                                        sum J, 0 (actor pass) */
  void *workspace;                   /* the pass's _workspace_bytes() bytes */
} wdb_td3_update_args;
/* 1 if a pass takes the shapes: those of wdb_ddpg_update_supported, both critics (and all
 * three targets) shaped alike, sigma, clip >= 0, and the pass's networks, gradient
 * accumulators and row tiles in one CTA's shared memory -- the critic pass holds five
 * networks and two critic gradient blocks.  No CUDA call. */
int wdb_td3_critic_update_supported(const wdb_td3_update_args *update);
long long wdb_td3_critic_update_workspace_bytes(const wdb_td3_update_args *update);  /* -1: unsupported */
int wdb_td3_actor_update_supported(const wdb_td3_update_args *update);
long long wdb_td3_actor_update_workspace_bytes(const wdb_td3_update_args *update);   /* -1: unsupported */
/* cudaErrorInvalidValue without launching if unsupported or a required pointer is NULL. */
int wdb_td3_critic_update(void *stream, const wdb_td3_update_args *update);
int wdb_td3_actor_update(void *stream, const wdb_td3_update_args *update);

/* One SAC update of one policy (Haarnoja et al. 2018) over the same ring and M loss rows as
 * wdb_ddpg_update, as two passes of two launches each (tile kernel + fixed-order reduction:
 * bit-reproducible).  The actor's head is Linear(H, 2A): mean mu, raw log-std clamped to
 * [log_std_min, log_std_max]; sigma = exp(log_std), u = mu + sigma * eps, a = scale * tanh(u) +
 * bias and
 *   log pi = sum_k [-eps_k^2 / 2 - log_std_k - log(2 pi) / 2 - 2 (log 2 - u_k - softplus(-2 u_k))]
 * (no action_scale term).  alpha = exp(*log_alpha), read on the device.
 * Critic pass (wdb_sac_critic_update), eps = critic_noise[g] at DDPG's bootstrap slot obs':
 *   R = the n-step return of DDPG bootstrapped with min(target_critic(obs', a'),
 *       target_critic2(obs', a')) - alpha log pi(a' | obs') (the actor, not a target actor),
 *   gradients of mse(Q1(obs, actions), R) + mse(Q2(obs, actions), R) into critic / critic2.
 * Actor pass (wdb_sac_actor_update), eps = actor_noise[g] at obs:
 *   the gradient of mean(alpha log pi(a | obs) - min(Q1, Q2)(obs, a)) into actor.gw / gb (ties
 *   of the minimum go to Q1; the critics' weights only carry it to their action inputs).
 * The critic pass reads actor, critic, critic2 and both target critics; the actor pass reads
 * actor, critic and critic2. */
typedef struct wdb_sac_update_args {
  int n_envs, n_agents, obs_dim, action_dim;   /* E, Np, F, A (the actor's head is 2A wide) */
  int capacity, cursor, n_step;      /* as wdb_ddpg_update_args */
  float gamma, action_scale, action_bias;
  float log_std_min, log_std_max;
  const float *log_alpha;            /* device [1] */
  const float *obs;                  /* [C, E, Np, F] */
  const float *actions;              /* [C, E, Np, A] */
  const float *rewards;              /* [C, E, Np] */
  const int *done;                   /* [C, E] */
  const float *critic_noise;         /* [valid, E * Np, A] standard normal, window order */
  const float *actor_noise;          /* [valid, E * Np, A] */
  wdb_ddpg_net actor, critic, critic2;          /* gradients: actor (actor pass), critics */
  wdb_ddpg_net target_critic, target_critic2;   /* the critic's shape */
  float *q1_values, *q2_values, *returns;       /* critic pass out [valid, E * Np], or NULL */
  float *log_probs;                  /* actor pass out [valid, E * Np], or NULL */
  double *sums;                      /* out [4]: sum (Q1 - R)^2, sum (Q2 - R)^2 (critic pass),
                                        sum min(Q1, Q2), sum log pi (actor pass) */
  void *workspace;                   /* the pass's _workspace_bytes() bytes */
} wdb_sac_update_args;
/* 1 if a pass takes the shapes: those of wdb_ddpg_update_supported with the actor's head 2A
 * wide (so A <= 32), both critics and their targets shaped alike, log_std_min <= log_std_max,
 * and the pass's networks, gradient accumulators and row tiles in one CTA's shared memory (the
 * critic pass holds the actor and four critics and two critic gradient blocks).  No CUDA
 * call. */
int wdb_sac_critic_update_supported(const wdb_sac_update_args *update);
long long wdb_sac_critic_update_workspace_bytes(const wdb_sac_update_args *update);  /* -1: unsupported */
int wdb_sac_actor_update_supported(const wdb_sac_update_args *update);
long long wdb_sac_actor_update_workspace_bytes(const wdb_sac_update_args *update);   /* -1: unsupported */
/* cudaErrorInvalidValue without launching if unsupported or a required pointer is NULL. */
int wdb_sac_critic_update(void *stream, const wdb_sac_update_args *update);
int wdb_sac_actor_update(void *stream, const wdb_sac_update_args *update);

/* Replay buffer: the same ring made long (capacity >= n_step + 1 slots of which `filled` hold
 * data, the oldest at physical slot `oldest`), and each of the five passes above over B
 * uniformly sampled n-step windows instead of every window of the ring.
 *
 * wdb_replay_sample_windows writes, for g < n_windows, windows[g] = {(oldest + k) mod capacity,
 * n}: a logical window start k uniform in [0, filled - n_step - 1] and an agent row n uniform
 * in [0, n_rows), n_rows = E * Np.  A window is the logical slots k .. k + n_step, so none
 * crosses the seam between the newest and the oldest data.  The draws are Philox4x32-10 with
 * key `seed` and counter (counter, g): no RNG state, the same (seed, counter) gives the same
 * windows.  A 32-bit draw x is reduced to [0, range) as the high word of x * range, so a value's
 * probability differs from 1 / range by less than 2^-32 (relative bias <= range / 2^32).
 * cudaErrorInvalidValue without launching unless n_step >= 1, n_step + 1 <= filled <= capacity,
 * 0 <= oldest < capacity, n_rows >= 1 and n_windows >= 1.  One launch. */
int wdb_replay_sample_windows(void *stream, int *windows /* out [n_windows][2] */, int n_windows,
                              unsigned long long seed, unsigned long long counter, int oldest,
                              int filled, int capacity, int n_step, int n_rows);

/* The loss rows of a *_sampled pass: row g is the window of agent row windows[g][1] that starts
 * at physical slot s = windows[g][0]; slot(j) = (s + j) mod capacity.  Observation and action
 * at slot(0), rewards and done flags at slot(0 .. n_step - 1), the bootstrap observation at
 * slot(n_step), and
 *   R = r_0 + (1 - d_0) gamma (r_1 + ... (1 - d_{n_step - 1}) gamma * bootstrap)
 * in the float32 operation order of a regular (not the last) window of the ring passes; there
 * is no last-window rule.  M = B = n_windows: the means, 2 / M, -1 / M, `sums` and the optional
 * per-row outputs ([B]) are those of the ring passes with that M, the noise inputs are [B, A],
 * and `cursor` of the args struct is not read.  A window may appear more than once; each
 * appearance is a loss row.  Every windows[g][0] must lie in [0, capacity) and windows[g][1] in
 * [0, E * Np): they are not checked on the device.  Bit-reproducible as the ring passes. */
typedef struct wdb_replay_windows {
  const int *windows;                /* device [B][2] */
  int n_windows;                     /* B >= 1 */
} wdb_replay_windows;
/* _sampled_supported: the ring pass's conditions without the one on cursor, capacity >= n_step
 * + 1 and n_windows >= 1.  The workspace depends on n_windows. */
int wdb_ddpg_update_sampled_supported(const wdb_ddpg_update_args *update, int n_windows);
long long wdb_ddpg_update_sampled_workspace_bytes(const wdb_ddpg_update_args *update, int n_windows);
int wdb_ddpg_update_sampled(void *stream, const wdb_ddpg_update_args *update,
                            const wdb_replay_windows *windows);
int wdb_td3_critic_update_sampled_supported(const wdb_td3_update_args *update, int n_windows);
long long wdb_td3_critic_update_sampled_workspace_bytes(const wdb_td3_update_args *update, int n_windows);
int wdb_td3_critic_update_sampled(void *stream, const wdb_td3_update_args *update,
                                  const wdb_replay_windows *windows);
int wdb_td3_actor_update_sampled_supported(const wdb_td3_update_args *update, int n_windows);
long long wdb_td3_actor_update_sampled_workspace_bytes(const wdb_td3_update_args *update, int n_windows);
int wdb_td3_actor_update_sampled(void *stream, const wdb_td3_update_args *update,
                                 const wdb_replay_windows *windows);
int wdb_sac_critic_update_sampled_supported(const wdb_sac_update_args *update, int n_windows);
long long wdb_sac_critic_update_sampled_workspace_bytes(const wdb_sac_update_args *update, int n_windows);
int wdb_sac_critic_update_sampled(void *stream, const wdb_sac_update_args *update,
                                  const wdb_replay_windows *windows);
int wdb_sac_actor_update_sampled_supported(const wdb_sac_update_args *update, int n_windows);
long long wdb_sac_actor_update_sampled_workspace_bytes(const wdb_sac_update_args *update, int n_windows);
int wdb_sac_actor_update_sampled(void *stream, const wdb_sac_update_args *update,
                                 const wdb_replay_windows *windows);

/* One double-DQN update of one policy (van Hasselt et al. 2016; n-step returns, Huber loss as
 * Mnih et al. 2015) over B sampled windows of the replay ring, as wdb_*_update_sampled read
 * them.  Per loss row g (window start slot s, agent row n) with obs at slot(0), the int32
 * action a at slot(0) and the bootstrap obs' at slot(n_step):
 *   boot = double_q ? target(obs')[argmax_a' online(obs')] : max_a' target(obs')
 *          (argmax: the first maximum),
 *   R    = r_0 + m_0 gamma (r_1 + ... m_{n_step - 1} gamma * boot), m_j = (done_j == 0),
 *          in the float32 operation order of the sampled passes (every non-zero done flag is
 *          terminal: MountainCar's 2 at the goal as well),
 *   loss = (1/B) sum_g huber(online(obs)[a] - R, delta),
 * and its gradient, clamp(Q - R, -delta, delta) / B in column a, back through the online
 * network into q.gw / gb.  Networks: hidden Linear + ReLU layers and a raw Linear head of A
 * outputs; target shaped as q.  Per-CTA partials summed in a fixed order by a second launch:
 * bit-reproducible.  Two launches.  The sums are Huber and Q only: they go through the fixed-order
 * reduction the DDPG passes use, which carries two doubles; the mean return comes from the
 * `returns` output when it is asked for. */
typedef struct wdb_dqn_update_args {
  int n_envs, n_agents, obs_dim, n_actions;   /* E, Np, F, A */
  int capacity, n_step;              /* ring slots C, n-step horizon (n_step + 1 <= C) */
  float gamma, huber_delta;          /* delta > 0 */
  int double_q;                      /* 0: bootstrap with max_a' target(obs') */
  const float *obs;                  /* [C, E, Np, F] */
  const int *actions;                /* [C, E, Np, 1] */
  const float *rewards;              /* [C, E, Np] */
  const int *done;                   /* [C, E] */
  wdb_ddpg_net q, target_q;          /* gradients: q; the target has q's shape */
  float *q_values, *returns;         /* out [B]: Q(obs, a) and R, or NULL */
  double *sums;                      /* out [2]: sum huber(Q - R), sum Q(obs, a) */
  void *workspace;                   /* wdb_dqn_update_sampled_workspace_bytes() bytes */
} wdb_dqn_update_args;
/* 1 if the shapes are supported: 0..3 hidden layers of width 1..64, 1 <= A <= 64, F <= 63, E, Np
 * >= 1, 1 <= n_step, n_step + 1 <= capacity, delta > 0, n_windows >= 1, and both networks, the
 * gradient accumulators and the row tiles in one CTA's shared memory.  No CUDA call. */
int wdb_dqn_update_sampled_supported(const wdb_dqn_update_args *update, int n_windows);
long long wdb_dqn_update_sampled_workspace_bytes(const wdb_dqn_update_args *update, int n_windows);
/* cudaErrorInvalidValue without launching if unsupported or a required pointer is NULL. */
int wdb_dqn_update_sampled(void *stream, const wdb_dqn_update_args *update,
                           const wdb_replay_windows *windows);

/* wdb_dqn_update_sampled with importance-sampling weights w [B] (wdb_per_sample_windows):
 *   loss = (1/B) sum_g w_g huber(Q_g - R_g, delta), head gradient w_g clamp(Q - R, -delta,
 *   delta) / B in column a, sums[0] = sum_g w_g huber(Q_g - R_g), sums[1] = sum Q(obs, a).
 * The weight multiplies the clamped difference before the 1 / B and the Huber value before the
 * sum, so all weights 1 reproduce wdb_dqn_update_sampled bit for bit.  Same shapes, workspace,
 * reduction and launch count (two). */
int wdb_dqn_update_prioritized_supported(const wdb_dqn_update_args *update, int n_windows);
long long wdb_dqn_update_prioritized_workspace_bytes(const wdb_dqn_update_args *update,
                                                     int n_windows);
/* cudaErrorInvalidValue without launching if unsupported or a required pointer (weights
 * included) is NULL. */
int wdb_dqn_update_prioritized(void *stream, const wdb_dqn_update_args *update,
                               const wdb_replay_windows *windows, const float *weights);

/* One quantile-regression DQN update (Dabney et al. 2018) over B sampled windows, read as
 * wdb_dqn_update_sampled reads them.  The networks' head has A * N outputs (n_actions = A,
 * n_quantiles = N); column a * N + i is quantile i of action a.  Per loss row g with action a:
 *   theta_i = online(obs)[a, i],  tau_i = (2 i + 1) / (2 N),
 *   a*      = the first argmax over actions of sum_j online(obs')[., j] (double_q) or of
 *             sum_j target(obs')[., j],
 *   T_j     = DQN's n-step recursion (float32, every non-zero done terminal) on
 *             target(obs')[a*, j],
 *   loss_g  = (1/N) sum_i sum_j |tau_i - 1{u_ij < 0}| huber(u_ij, kappa) / kappa,
 *             u_ij = T_j - theta_i, kappa = huber_delta,
 *   loss    = (1/B) sum_g w_g loss_g,  w_g = weights[g], or 1 when weights is NULL,
 * and its gradient, -w_g / (kappa N B) sum_j |tau_i - 1{u_ij < 0}| clamp(u_ij, -kappa, kappa)
 * in column a * N + i (the sum over j in order), back through the online network into q.gw /
 * gb.  sums[0] = sum_g w_g loss_g, sums[1] = sum_g mean_i theta_i; the optional outputs [B] are
 * q_values = mean_i theta_i and returns = mean_j T_j.  The weight multiplies a row's gradient
 * and loss once each, so unit weights reproduce the unweighted pass bit for bit.  Per-CTA
 * partials summed in a fixed order by a second launch: bit-reproducible.  Two launches.
 * Supported: the shapes of wdb_dqn_update_sampled_supported with n_quantiles >= 1 and the head
 * A * N <= 64.  No CUDA call. */
int wdb_qr_dqn_update_sampled_supported(const wdb_dqn_update_args *update, int n_quantiles,
                                        int n_windows);
long long wdb_qr_dqn_update_sampled_workspace_bytes(const wdb_dqn_update_args *update,
                                                    int n_quantiles, int n_windows);
/* cudaErrorInvalidValue without launching if unsupported or a required pointer is NULL. */
int wdb_qr_dqn_update_sampled(void *stream, const wdb_dqn_update_args *update, int n_quantiles,
                              const wdb_replay_windows *windows, const float *weights);

/* One implicit quantile network update (IQN; Dabney, Ostrovski, Silver & Munos 2018) over B
 * sampled windows, read as wdb_dqn_update_sampled reads them.  q / target_q are the trunk psi
 * (their hidden Linear + ReLU layers, at least one, width H) and a raw head Linear(H, A); the
 * tau embedding of each is phi(tau) = ReLU(E f(tau) + e), E [H, n_cos], with the cosine
 * features f_c(tau) = cos(float(pi * c) * tau), c = 0 .. n_cos - 1 (float32 multiply, cosf).
 * Z_tau(x, .) = head(psi(x) * phi(tau)).  Per loss row g with action a, levels tau_i = taus[g][i]
 * (i < N) and tau'_j = taus[g][N + j] (j < N'):
 *   c-bar   = mean_k phi(tau~_k) over the K midpoints tau~_k = (2k + 1) / (2K), of the online
 *             embedding (double_q) or the target one; Q-bar(x, .) = head(psi(x) * c-bar),
 *   a*      = the first argmax of Q-bar of online(obs') (double_q) or of target(obs'),
 *   theta_i = Z_tau_i(obs)[a] (online),  T_j = DQN's n-step recursion (float32, every non-zero
 *             done terminal) on the target's Z_tau'_j(obs')[a*],
 *   loss_g  = (1/N') sum_i sum_j |tau_i - 1{u_ij < 0}| huber(u_ij, kappa) / kappa,
 *             u_ij = T_j - theta_i, kappa = huber_delta,
 *   loss    = (1/B) sum_g w_g loss_g,  w_g = weights[g], or 1 when weights is NULL,
 * and its gradient, d loss / d theta_i = -w_g / (kappa N' B) sum_j |tau_i - 1{u_ij < 0}|
 * clamp(u_ij, -kappa, kappa) (the sum over j in order), back through the head (summed over the
 * row's pairs), the merge (d psi summed over i in order) and the embedding (through its ReLU,
 * the cosine features recomputed) into q.gw / gb and embed_gw / gb.  sums[0] = sum_g w_g
 * loss_g, sums[1] = sum_g mean_i theta_i; the optional outputs [B] are q_values = mean_i
 * theta_i and returns = mean_j T_j.  The weight multiplies a row's gradient and loss once each,
 * so unit weights reproduce the unweighted pass bit for bit.  Per-CTA partials summed in a fixed
 * order by a second launch: bit-reproducible.  Two launches. */
typedef struct wdb_iqn_args {
  int n_cos, n_tau, n_tau_prime, n_quantile_samples;   /* n_cos, N, N', K */
  const float *taus;                 /* [B, N + N']: each row's tau_i, then its tau'_j */
  wdb_ddpg_net embed, target_embed;  /* the tau embeddings, n_hidden = 0: w[0] = E [H, n_cos],
                                        b[0] = e [H]; gw[0] / gb[0] the online one's gradients */
} wdb_iqn_args;
/* Supported: the shapes of wdb_dqn_update_sampled_supported with at least one hidden layer,
 * 1 <= n_cos, N, N' <= 64, 1 <= K <= 256, and both Q networks, both embeddings, both gradient
 * blocks and the row tiles in one CTA's shared memory.  No CUDA call. */
int wdb_iqn_update_sampled_supported(const wdb_dqn_update_args *update, const wdb_iqn_args *iqn,
                                     int n_windows);
long long wdb_iqn_update_sampled_workspace_bytes(const wdb_dqn_update_args *update,
                                                 const wdb_iqn_args *iqn, int n_windows);
/* cudaErrorInvalidValue without launching if unsupported or a required pointer is NULL. */
int wdb_iqn_update_sampled(void *stream, const wdb_dqn_update_args *update,
                           const wdb_iqn_args *iqn, const wdb_replay_windows *windows,
                           const float *weights);

/* One categorical DQN update (C51; Bellemare, Dabney & Munos 2017) over B sampled windows, read
 * as wdb_dqn_update_sampled reads them.  The networks' head has A * N outputs (n_actions = A,
 * n_atoms = N); column a * N + j is the logit of atom j of action a.  support [N] (device) holds
 * the atoms z_0 < ... < z_{N-1}, delta_z > 0 their spacing.  Per loss row g with action a, in
 * float32 (sums "over the row": lane k of the row's 16 threads takes j = k, k + 16, ... in
 * order, then the 16 lanes are combined by an xor butterfly; every lane gets the same bits):
 *   Q(x, c)  = q / s over the row, e_j = expf(y_j - max_j y_j), s = sum e_j, q = sum fmaf(z_j,
 *              e_j, .), y = the logits of action c at x,
 *   a*       = the first argmax over c of Q(obs', c) of online (double_q) or target,
 *   p'_j     = e_j / s of target(obs')[a*],
 *   Tz_j     = DQN's n-step recursion (float32, every non-zero done terminal) on z_j, then
 *              fminf(fmaxf(., z_0), z_{N-1}),
 *   m_i      = sum_j (j in order) fmaf(clip(1 - |Tz_j - z_i| / delta_z, 0, 1), p'_j, .),
 *   p_i      = expf(l_i - max l) / s of the online logits l = online(obs)[a],
 *   loss_g   = -sum_i m_i log_softmax(l)_i (in float64),
 *   loss     = (1/B) sum_g w_g loss_g,  w_g = weights[g], or 1 when weights is NULL,
 * and its gradient d loss / d l_i = ((p_i * sum_k m_k - m_i) * w_g) * (1/B) (sum_k m_k over the
 * row; not assumed to be 1) in column a * N + i, back through the online network into q.gw /
 * gb.  sums[0] = sum_g w_g loss_g, sums[1] = sum_g Q-bar_g; the optional outputs [B] are
 * q_values = Q-bar = sum_i z_i p_i and returns = R-bar = sum_i z_i m_i (float64 sums, stored
 * as float32).  huber_delta is not read.  The weight multiplies a row's gradient and loss once
 * each, so unit weights reproduce the unweighted pass bit for bit.  Per-CTA partials summed in
 * a fixed order by a second launch: bit-reproducible.  Two launches.
 * Supported: the shapes of wdb_dqn_update_sampled_supported (the head A * N may exceed 64) with
 * 2 <= N <= 64, and both networks, the gradient block and the row tiles in one CTA's shared
 * memory.  No CUDA call. */
int wdb_c51_update_sampled_supported(const wdb_dqn_update_args *update, int n_atoms,
                                     int n_windows);
long long wdb_c51_update_sampled_workspace_bytes(const wdb_dqn_update_args *update,
                                                 int n_atoms, int n_windows);
/* cudaErrorInvalidValue without launching if unsupported, a required pointer is NULL or
 * delta_z <= 0. */
int wdb_c51_update_sampled(void *stream, const wdb_dqn_update_args *update, int n_atoms,
                           const float *support, float delta_z,
                           const wdb_replay_windows *windows, const float *weights);

/* Action masks (DQN and C51).  action_mask [C, E, Np, A] (float32, non-zero = valid) is the
 * ring's mask array beside obs: the row at a window's slot(n_step) is obs' own mask.  The
 * bootstrap's a* -- the double-Q argmax of online(obs'), DQN's max_a' target(obs') and C51's
 * argmax of the expectation -- ranges over the valid actions of that row only; a row with no
 * valid action takes every action (the unmasked rule: the device can neither refuse it nor
 * report it without a host wait).  The loss row is unchanged: the action at slot(0) was chosen
 * under its own mask.  The mask is read by the bootstrap alone, and an all-ones mask gives the
 * unmasked pass's bits.  weights NULL: the uniform pass; else the importance-weighted one.
 * Shapes, workspace, sums, outputs and launches (two) are the unmasked pass's. */
int wdb_dqn_update_masked_supported(const wdb_dqn_update_args *update, int n_windows);
long long wdb_dqn_update_masked_workspace_bytes(const wdb_dqn_update_args *update,
                                                int n_windows);
/* wdb_dqn_update_sampled / _prioritized with the masked bootstrap.  cudaErrorInvalidValue
 * without launching if unsupported or a required pointer (action_mask included) is NULL. */
int wdb_dqn_update_masked(void *stream, const wdb_dqn_update_args *update,
                          const wdb_replay_windows *windows, const float *weights,
                          const float *action_mask);
int wdb_c51_update_masked_supported(const wdb_dqn_update_args *update, int n_atoms,
                                    int n_windows);
long long wdb_c51_update_masked_workspace_bytes(const wdb_dqn_update_args *update, int n_atoms,
                                                int n_windows);
/* wdb_c51_update_sampled with the masked a*.  cudaErrorInvalidValue without launching if
 * unsupported, a required pointer (action_mask included) is NULL or delta_z <= 0. */
int wdb_c51_update_masked(void *stream, const wdb_dqn_update_args *update, int n_atoms,
                          const float *support, float delta_z, const wdb_replay_windows *windows,
                          const float *weights, const float *action_mask);

/* Action branching (Tavakoli, Pardo & Kormushev 2018): one Q head per action dimension of a
 * MultiDiscrete space on a shared trunk.  Heads d = 0 .. D-1 have sizes A_d and offsets
 * o_d = A_0 + ... + A_{d-1}; the network's raw head has A = sum_d A_d outputs and Q_d(s, .) is
 * columns o_d .. o_d + A_d - 1.  Actions are laid out [rows, D]: one int32 per head. */
typedef struct wdb_q_branches {
  int n_heads;                       /* D, 1 .. 16 */
  int sizes[16];                     /* A_d >= 1 for d < D; the rest are not read */
} wdb_q_branches;

/* Epsilon-greedy per head: row r's head d applies wdb_sample_epsilon_greedy's rule to Q_d with
 * ONE Philox block on stream r at offset o_r + d (o_r the row's offset), or with the words
 * (x, y) = words[r][d] ([n_rows][D][2], test hook; no RNG state read or advanced); the row's
 * offset then advances by D.  Each head explores on its own with probability epsilon.
 * q_values [n_rows, A], actions [n_rows, D].  At D = 1 the actions and offsets are
 * wdb_sample_epsilon_greedy's bit for bit.  One launch.  cudaErrorInvalidValue unless
 * 0 <= epsilon <= 1 and the branches are valid (1 <= D <= 16, every A_d >= 1). */
int wdb_sample_epsilon_greedy_branching(void *stream, void *rng_state, const float *q_values,
                                        const wdb_q_branches *branches, int *actions,
                                        long long n_rows, float epsilon,
                                        const unsigned int *words);

/* One branching double-DQN update over B sampled windows, read as wdb_dqn_update_sampled reads
 * them, with update->n_actions = A and actions [C, E, Np, D].  Per window g with the D actions
 * a_d at slot(0), every float32 operation in ascending d:
 *   a*_d   = the first argmax of online_d(obs') (double_q),
 *   boot_d = target_d(obs')[a*_d]  (double_q) or max target_d(obs'),
 *   boot   = (sum_d boot_d) / D (the mean target of BDQ),
 *   R      = DQN's n-step recursion from boot (every non-zero done flag terminal),
 *   loss   = (1/B) sum_g w_g (1/D) sum_d huber(Q_d(obs, a_d) - R, delta),
 * and its gradient w_g clamp(Q_d - R, -delta, delta) * (float)(1 / (B D)) in column o_d + a_d,
 * back through the online network into q.gw / gb (w_g = weights[g], or 1 without weights).  An
 * action outside [0, A_d) contributes nothing.  sums[0] = sum_g w_g (1/D) sum_d huber,
 * sums[1] = sum_g Q-bar_g; the optional outputs [B] are q_values = Q-bar_g = (sum_d
 * Q_d(obs, a_d)) / D and returns = R.  Every divide by D is exact at D = 1, so one head gives
 * wdb_dqn_update_sampled's / _prioritized's bits.  Per-CTA partials summed in a fixed order by
 * a second launch: bit-reproducible.  Two launches.
 * Supported: the shapes of wdb_dqn_update_sampled_supported with 1 <= D <= 16, every A_d >= 1
 * and sum_d A_d = A <= 64.  No CUDA call. */
int wdb_branching_dqn_update_sampled_supported(const wdb_dqn_update_args *update,
                                               const wdb_q_branches *branches, int n_windows);
long long wdb_branching_dqn_update_sampled_workspace_bytes(const wdb_dqn_update_args *update,
                                                           const wdb_q_branches *branches,
                                                           int n_windows);
/* cudaErrorInvalidValue without launching if unsupported or a required pointer is NULL. */
int wdb_branching_dqn_update_sampled(void *stream, const wdb_dqn_update_args *update,
                                     const wdb_q_branches *branches,
                                     const wdb_replay_windows *windows);
/* The importance-weighted form (weights [B], wdb_per_sample_windows): the same shapes,
 * workspace, sums and launches.  Unit weights reproduce the uniform pass bit for bit. */
int wdb_branching_dqn_update_prioritized_supported(const wdb_dqn_update_args *update,
                                                   const wdb_q_branches *branches,
                                                   int n_windows);
long long wdb_branching_dqn_update_prioritized_workspace_bytes(const wdb_dqn_update_args *update,
                                                               const wdb_q_branches *branches,
                                                               int n_windows);
/* cudaErrorInvalidValue without launching if unsupported or a required pointer (weights
 * included) is NULL. */
int wdb_branching_dqn_update_prioritized(void *stream, const wdb_dqn_update_args *update,
                                         const wdb_q_branches *branches,
                                         const wdb_replay_windows *windows,
                                         const float *weights);

/* Dueling head (Wang et al. 2016, the mean combine) of a DQN or C51 network, and its fold into
 * the plain MLP head the passes above run.  The head reads the trunk output h (width H) through
 * two streams, each with one hidden Linear(H, S) + ReLU when S > 0 and none when S = 0 (the
 * output layer then reads h):
 *   V = value(h) [N],  Adv = advantage(h) [A N],
 *   out[a N + j] = V_j + Adv[a N + j] - (1/A) sum_c Adv[c N + j]   (N = 1: DQN, N atoms: C51).
 * The combine is linear in the output layers, so the head is exactly this folded network:
 *   hidden (S > 0): w = [value_hw; adv_hw] [2S, H], b = [value_hb; adv_hb] [2S],
 *   output, K = 2S: ow[a N + j] = [value_ow[j] | adv_ow[a N + j] - m_j], m_j = (1/A) sum_c
 *                   adv_ow[c N + j] ([A N, 2S]),
 *           K = H (S = 0): ow[a N + j] = value_ow[j] + (adv_ow[a N + j] - m_j) ([A N, H]),
 *   ob[a N + j] = value_ob[j] + (adv_ob[a N + j] - m'_j), m'_j the same mean of adv_ob.
 * Means are float32 sums over c = 0 .. A - 1 in order, divided by A, so a fold or an unfold is
 * bit-reproducible.  Row-major nn.Linear layouts throughout ([out, in] weights). */
typedef struct wdb_dueling_head {
  int n_actions, n_atoms, in_dim, stream_dim;   /* A, N, H, S (0: no stream hidden layer) */
  const float *value_hw, *value_hb;  /* value stream hidden Linear(H, S) (S > 0; else unread) */
  const float *value_ow, *value_ob;  /* value stream output Linear(S or H, N) */
  const float *adv_hw, *adv_hb;      /* advantage stream hidden Linear(H, S) (S > 0) */
  const float *adv_ow, *adv_ob;      /* advantage stream output Linear(S or H, A N) */
  float *value_ghw, *value_ghb, *value_gow, *value_gob;   /* stream gradients, the shapes above */
  float *adv_ghw, *adv_ghb, *adv_gow, *adv_gob;           /* (written by the unfold) */
  float *hw, *hb, *ow, *ob;          /* folded layers (written by the fold; hw, hb when S > 0) */
  const float *ghw, *ghb, *gow, *gob;  /* their gradients (read by the unfold; ghw, ghb: S > 0) */
} wdb_dueling_head;
/* 1 if the fold / unfold take the shape: A, N, H >= 1, S >= 0, and every folded layer below
 * 2^31 elements.  No CUDA call. */
int wdb_dueling_fold_supported(const wdb_dueling_head *head);
int wdb_dueling_unfold_grads_supported(const wdb_dueling_head *head);
/* Writes head's folded layers from its stream parameters and, when target is not NULL, the
 * target's from its own (same shape; its gradient pointers are not read).  One launch.
 * cudaErrorInvalidValue without launching if unsupported, the shapes differ or a required
 * pointer is NULL. */
int wdb_dueling_fold(void *stream, const wdb_dueling_head *head, const wdb_dueling_head *target);
/* Writes the stream parameters' gradients from the folded layers' gradients, through the
 * transpose of the fold:
 *   hidden: value_ghw / ghb = rows 0 .. S - 1 of ghw / ghb, adv_ghw / ghb = rows S .. 2S - 1,
 *   value_gow[j][k] = sum_a gow[a N + j][k]   (k < S; all of row k when S = 0), value_gob alike,
 *   adv_gow[a N + j][k] = g[a N + j][k] - (1/A) sum_c g[c N + j][k], g = gow's columns S .. 2S-1
 *                         (S > 0) or all of gow (S = 0), adv_gob alike from gob.
 * Sums over a and c in order.  One launch.  cudaErrorInvalidValue without launching if
 * unsupported or a required pointer is NULL. */
int wdb_dueling_unfold_grads(void *stream, const wdb_dueling_head *head);

/* Noisy networks (Fortunato et al. 2018, factorized Gaussian noise) of a DQN or C51 head.  A
 * noisy layer of in_dim inputs and out_dim outputs has parameters mu_W, sigma_W [out, in] and
 * mu_b, sigma_b [out]; with the noise vectors fi = f(eps_in) [in], fo = f(eps_out) [out],
 * f(x) = sgn(x) sqrt(|x|), its effective layer is
 *   W[j][k] = fmaf(sigma_W[j][k], fo[j] * fi[k], mu_W[j][k]),  b[j] = fmaf(sigma_b[j], fo[j], mu_b[j]).
 * The noise element: eps = u32x2_to_normal of two words of Philox4x32-10 with key `seed` (the
 * trainer seed) at the counter
 *   (count mod 2^32, 0x4E000000 | domain << 16 | (count >> 32) mod 2^16, row,
 *    layer << 16 | e >> 1),
 * words (x, y) for an even element e and (z, w) for an odd one.  domain 0 is the update (count:
 * the update number; row 0 the online network's sample, row 1 the target's), domain 1 acting
 * (count: the policy's acting step; row: the env row).  e < in_dim is eps_in[e], e >= in_dim
 * eps_out[e - in_dim]; layer numbers the head's noisy layers in module order.  The counter's
 * second word is at least 0x4E000000, so no draw of wdb_replay_sample_windows,
 * wdb_per_sample_windows (counter (n, g): second word n >> 32) or of the sampler's per-env and
 * reset-pool streams (offset (o, o >> 32, stream, stream >> 32)) coincides with a noise draw
 * below 2^56 draws. */
#define WDB_NOISY_MAX_LAYERS 4
typedef struct wdb_noisy_layer {
  int in_dim, out_dim;               /* in_dim + out_dim <= 2^17 */
  const float *weight_mu, *weight_sigma;   /* [out, in] */
  const float *bias_mu, *bias_sigma;       /* [out] */
  float *noise_in, *noise_out;       /* f(eps_in) [rows, in], f(eps_out) [rows, out] */
  float *weight, *bias;              /* the effective W [out, in], b [out] (materialize) */
  const float *grad_weight, *grad_bias;    /* dW, db (read by the grads) */
  float *grad_weight_mu, *grad_weight_sigma, *grad_bias_mu, *grad_bias_sigma;   /* (written) */
} wdb_noisy_layer;
typedef struct wdb_noisy_net {
  int n_layers;                      /* 1 .. WDB_NOISY_MAX_LAYERS */
  wdb_noisy_layer layer[WDB_NOISY_MAX_LAYERS];
} wdb_noisy_net;
/* 1 if the noisy kernels take the shape: 1 <= n_layers <= 4, every in_dim, out_dim >= 1,
 * in_dim + out_dim <= 2^17 and in_dim * out_dim < 2^31.  No CUDA call. */
int wdb_noisy_supported(const wdb_noisy_net *net);
/* Writes f(eps) of rows row0 .. row0 + n_rows - 1 of (domain, count): layer l's noise_in[r][k]
 * and noise_out[r][j], r = 0 .. n_rows - 1 for counter row row0 + r.  Only the noise pointers
 * are read.  One launch.  cudaErrorInvalidValue without launching if unsupported, n_rows < 1,
 * domain is not 0 or 1, or a noise pointer is NULL. */
int wdb_noisy_draw(void *stream, const wdb_noisy_net *net, unsigned long long seed, int domain,
                   unsigned long long count, int row0, int n_rows);
/* The update's samples: for the online net (row 0) and, when target is not NULL, the target (row
 * 1) of update `update`, writes f(eps) into noise_in / noise_out ([1, in], [1, out]) and the
 * effective layers into weight / bias.  One launch.  cudaErrorInvalidValue without launching if
 * unsupported, the shapes differ or a pointer it reads or writes is NULL. */
int wdb_noisy_materialize(void *stream, const wdb_noisy_net *online, const wdb_noisy_net *target,
                          unsigned long long seed, unsigned long long update);
/* From the effective layers' gradients dW, db and the noise vectors materialize wrote:
 *   grad_weight_mu = dW, grad_weight_sigma[j][k] = dW[j][k] * (fo[j] * fi[k]),
 *   grad_bias_mu = db, grad_bias_sigma[j] = db[j] * fo[j]   (float32 products, no sums).
 * One launch.  cudaErrorInvalidValue without launching if unsupported or a pointer is NULL. */
int wdb_noisy_grads(void *stream, const wdb_noisy_net *net);

/* Prioritized replay (Schaul et al. 2016, proportional) over the replay ring's n-step windows.
 * One float32 leaf per (physical slot s, agent row n), leaf s * n_rows + n: p^alpha of the
 * window that starts at slot s for agent row n (windows[g] = {s, n} as above), and 0 exactly
 * when that window is not valid -- its logical start k (slots after the oldest) is not in
 * [0, filled - n_step - 1].  Over the leaves a sum tree of fan-out 32 with float64 nodes, level
 * by level from the leaves' parents up to the root; a node is its (up to 32, zero-padded)
 * children summed pairwise, v[i] += v[i + h] for h = 16, 8, 4, 2, 1.  Every write repairs the
 * paths above the leaves it touched, one launch per tree level, by recomputing each node from
 * its children, so the tree is always a pure function of the leaves (bit for bit what a fresh
 * build gives).  p_max is the running maximum of the priorities (|delta| + epsilon) written,
 * 1 at the start; new windows enter at p_max^alpha.  The leaf count capacity * n_rows must be
 * below 2^31. */
typedef struct wdb_per_store {
  int capacity, n_rows, n_step;      /* ring slots C (>= n_step + 1), E * Np, n-step horizon */
  float alpha, epsilon;              /* alpha in [0, 1], epsilon > 0 */
  float *leaves;                     /* device [C * n_rows], zeros at the start */
  double *nodes;                     /* device [wdb_per_nodes(C * n_rows)], zeros at the start */
  float *p_max;                      /* device [1], 1 at the start */
} wdb_per_store;
/* The float64 nodes / the levels of the tree over n_leaves leaves; -1 unless 1 <= n_leaves <
 * 2^31.  No CUDA call. */
long long wdb_per_nodes(long long n_leaves);
int wdb_per_levels(long long n_leaves);
/* After each rollout of T slots, given the ring's cursor and fill level before and after it
 * (T = cursor_after - cursor_before mod C): the leaves of the starts that have just become
 * valid get p_max^alpha, those of the newest n_step slots (the slots the rollout overwrote among
 * them) get 0, then the touched paths are repaired.  Needs 1 <= T, T + n_step <= C and
 * filled_after = min(C, filled_before + T).  1 + levels launches. */
int wdb_per_admit(void *stream, const wdb_per_store *store, int cursor_before, int filled_before,
                  int cursor_after, int filled_after);
/* B windows by stratified proportional sampling: row g draws u in [g S / B, (g + 1) S / B) (S:
 * the root, read on the device) as lo + U (hi - lo), U = (a >> 5 * 2^26 + b >> 6) / 2^53 from
 * the words a, b of Philox4x32-10 with key `seed` at counter (counter, g), and descends: the
 * children of a node are scanned in order with a running float64 prefix, the first with
 * positive mass whose prefix end exceeds u is entered and u drops by the prefix before it; if
 * rounding puts u at or past the node's total, the last child with positive mass is entered
 * (a zero-sum child never is).  Writes windows[g] = {s, n}, priorities[g] = the leaf p^alpha,
 * and, from a second one-CTA launch, weights[g] = (priorities[g] / min_g priorities)^-beta with
 * beta read from the device (the weights normalised by the batch's largest, as Dopamine and
 * Rainbow do).  The store must hold a valid window.  Two launches, no host wait. */
int wdb_per_sample_windows(void *stream, const wdb_per_store *store,
                           int *windows /* out [B][2] */, float *priorities /* out [B] */,
                           float *weights /* out [B] */, int n_windows,
                           unsigned long long seed, unsigned long long counter,
                           const float *beta /* device [1] */);
/* Writes (|q_values[g] - returns[g]| + epsilon)^alpha to the leaf of each window that is a
 * valid start of the ring (`oldest`, `filled` as wdb_replay_sample_windows; other rows are
 * skipped), raises p_max, and repairs the touched paths.  A window given twice keeps its larger
 * priority whatever the order.  A non-finite priority is taken as the largest float.
 * 2 + levels launches. */
int wdb_per_set_priorities(void *stream, const wdb_per_store *store, const int *windows,
                           int n_windows, const float *q_values, const float *returns,
                           int oldest, int filled);

/* Running observation statistics (per feature of a row-major [rows, F] float32 batch) and the
 * normalization they drive.  A moments record is rows of float64 [n, mean_0 .. mean_{F-1},
 * M2_0 .. M2_{F-1}] (M2 = the sum of squared deviations).  The running state is count
 * (device scalar), mean [F] and M2 [F] in float64, and the float32 shift [F] = mean and scale
 * [F] = 1 / sqrt(M2 / count + 1e-8) that the forwards read (count 0: shift 0, scale 1).
 * Merges are Chan et al.'s in a fixed order, with no float atomics: bit-reproducible.
 * 1 <= F <= 65536.  cudaErrorInvalidValue without launching on a bad shape or NULL pointer. */
/* float64 elements of the scratch the update and batch passes take for `rows` x F (-1: bad
 * shape). */
long long wdb_obs_moments_scratch_doubles(long long rows, int F);
/* Merges the batch x [rows, F] into the running state and rewrites shift and scale.  Two
 * launches (per-CTA Welford records over fixed row ranges into scratch, then one CTA merging
 * them in order), no host wait. */
int wdb_obs_moments_update(void *stream, const float *x, long long rows, int F, double *scratch,
                           double *count, double *mean, double *m2, float *shift, float *scale);
/* The batch's own moments as one record [2F + 1] (two launches): what each GPU contributes
 * before the records are gathered. */
int wdb_obs_moments_batch(void *stream, const float *x, long long rows, int F, double *scratch,
                          double *record);
/* Merges n_records (<= 512) records [n_records][2F + 1] in order into the running state and
 * rewrites shift and scale.  One launch. */
int wdb_obs_moments_merge(void *stream, const double *records, int n_records, int F,
                          double *count, double *mean, double *m2, float *shift, float *scale);
/* y [rows, F] = clamp((x - shift) * scale, -clip, clip) per feature (clip finite, > 0): a
 * rounded subtract, a rounded multiply, then the clamp.  One launch. */
int wdb_obs_normalize(void *stream, const float *x, float *y, long long rows, int F,
                      const float *shift, const float *scale, float clip);

/* The running discounted return of reward scaling (SB3 VecNormalize's return filter), forward
 * in time for every (env, agent) row i of rewards [T, E, Np] f32 and done [T, E] i32:
 *   ret = __fadd_rn(__fmul_rn(gamma, carry[i]), r[t][i]);  returns[t][i] = ret;
 *   carry[i] = done[t][env] > 0 ? 0 : ret.
 * carry [E, Np] f32 is read and left holding the return after step T - 1.  No FMA is
 * contracted, so a float32 restatement gives the same bits.  One launch, one thread per row.
 * cudaErrorInvalidValue without launching on a NULL pointer or T, n_envs or n_agents < 1. */
int wdb_discounted_return_scan(void *stream, const float *rewards, const int *done, int T,
                               int n_envs, int n_agents, float gamma, float *carry,
                               float *returns);

/* One discrete-action SAC update of one policy (Christodoulou 2019) over B sampled windows, read
 * as wdb_dqn_update_sampled reads them, as two passes of two launches each (a tile kernel and
 * the fixed-order reduction: bit-reproducible).  The actor and the four Q networks map F -> A
 * (hidden Linear + ReLU layers, a raw Linear head): the actor's head is the logits z of a
 * categorical policy, log pi = z - max z - log sum_a exp(z_a - max z) (a log-softmax), and each Q
 * network's head is A action values.  alpha = exp(*log_alpha), read on the device.  Every sum
 * over actions runs a = 0 .. A - 1 in order.
 * Critic pass (wdb_sac_discrete_critic_update_sampled), per loss row g with the int32 action a
 * at slot(0), obs at slot(0) and obs' at slot(n_step):
 *   V' = sum_a pi'_a (min(target_critic(obs'), target_critic2(obs'))_a - alpha log pi'_a),
 *        pi' = the actor's policy at obs' (no target actor),
 *   R  = DQN's n-step recursion on V' (float32, every non-zero done flag terminal),
 *   gradients of mse(critic(obs)[a], R) + mse(critic2(obs)[a], R) into critic / critic2.
 * Actor pass (wdb_sac_discrete_actor_update_sampled), with h_a = alpha log pi_a - min(critic(obs),
 *   critic2(obs))_a: the gradient of (1/B) sum_g sum_a pi_a h_a, d/dz_j = pi_j (h_j - sum_a pi_a
 *   h_a) / B, into actor.gw / gb (no critic gradient).
 * The critic pass reads actor, critic, critic2 and both target critics; the actor pass reads
 * actor, critic and critic2. */
typedef struct wdb_sac_discrete_update_args {
  int n_envs, n_agents, obs_dim, n_actions;   /* E, Np, F, A */
  int capacity, n_step;              /* ring slots C, n-step horizon (n_step + 1 <= C) */
  float gamma;
  const float *obs;                  /* [C, E, Np, F] */
  const int *actions;                /* [C, E, Np, 1] */
  const float *rewards;              /* [C, E, Np] */
  const int *done;                   /* [C, E] */
  const float *log_alpha;            /* device [1] */
  wdb_ddpg_net actor, critic, critic2;          /* gradients: actor (actor pass), critics */
  wdb_ddpg_net target_critic, target_critic2;   /* the critic's shape */
  float *q1_values, *q2_values, *returns;       /* critic pass out [B]: Q1(obs)[a], Q2(obs)[a],
                                                   R; or NULL */
  float *entropies;                  /* actor pass out [B]: -sum_a pi_a log pi_a, or NULL */
  double *sums;                      /* out [4]: sum (Q1 - R)^2, sum (Q2 - R)^2 (critic pass),
                                        sum_g sum_a pi_a min(Q1, Q2)_a, sum_g sum_a pi_a log pi_a
                                        (actor pass) */
  void *workspace;                   /* the pass's _workspace_bytes() bytes */
} wdb_sac_discrete_update_args;
/* 1 if a pass takes the shapes: 0..3 hidden layers of width 1..64 per network, the four Q
 * networks shaped alike, 2 <= A <= 64, F <= 63, E, Np >= 1, 1 <= n_step, n_step + 1 <= capacity,
 * n_windows >= 1, and the pass's networks, gradient blocks and row tiles in one CTA's shared
 * memory (the critic pass holds the actor, four Q networks and two gradient blocks).  No CUDA
 * call. */
int wdb_sac_discrete_critic_update_sampled_supported(const wdb_sac_discrete_update_args *update,
                                                     int n_windows);
long long wdb_sac_discrete_critic_update_sampled_workspace_bytes(
    const wdb_sac_discrete_update_args *update, int n_windows);   /* -1: unsupported */
int wdb_sac_discrete_actor_update_sampled_supported(const wdb_sac_discrete_update_args *update,
                                                    int n_windows);
long long wdb_sac_discrete_actor_update_sampled_workspace_bytes(
    const wdb_sac_discrete_update_args *update, int n_windows);   /* -1: unsupported */
/* cudaErrorInvalidValue without launching if unsupported or a required pointer is NULL. */
int wdb_sac_discrete_critic_update_sampled(void *stream, const wdb_sac_discrete_update_args *update,
                                           const wdb_replay_windows *windows);
int wdb_sac_discrete_actor_update_sampled(void *stream, const wdb_sac_discrete_update_args *update,
                                          const wdb_replay_windows *windows);

/* One TQC update of one policy (Kuznetsov et al. 2020, "Controlling Overestimation Bias with
 * Truncated Mixture of Continuous Distributional Quantile Critics") over B sampled windows, read
 * as wdb_sac_*_update_sampled read them, as two passes of two launches each (a tile kernel and
 * the fixed-order reduction: bit-reproducible).  The actor is SAC's squashed Gaussian
 * (wdb_sac_update_args: head 2A, the same sample and log pi); the two critics and their targets
 * map obs ++ action to N quantiles theta_m,i (hidden Linear + ReLU layers, a raw Linear(H, N)
 * head).  tau_i = (2i + 1) / (2N) in float32, K = 2 (N - n_drop), alpha = exp(*log_alpha) read
 * on the device, H(u) = u^2 / 2 for |u| <= 1 else |u| - 1/2.
 * Critic pass (wdb_tqc_critic_update_sampled), eps' = critic_noise[g] at obs' = obs at slot(n_step):
 *   a', log pi' = the actor's sample at obs' (no target actor),
 *   y_0 <= .. <= y_{K-1} = the K smallest of the 2N pooled atoms target_critic(obs', a') ++
 *       target_critic2(obs', a') (pooled index m N + j; ties to the lower index: a stable sort),
 *   T_k = the n-step return of the sampled passes bootstrapped with y_k - alpha log pi',
 *   loss = sum_g sum_m,i,k |tau_i - 1{u < 0}| H(u) / (B 2 N K),  u = T_k - theta_m,i(obs, a),
 *   its gradient d theta_m,i = -sum_k |tau_i - 1{u < 0}| clamp(u, -1, 1) / (B 2 N K) (each sum
 *   over k ascending) back through critic / critic2 into their gw / gb (the targets detached).
 * Actor pass (wdb_tqc_actor_update_sampled), eps = actor_noise[g] at obs: the gradient of
 *   (1/B) sum_g (alpha log pi - Qbar_g), Qbar_g = the mean of the 2N quantiles of both critics at
 *   (obs, a), into actor.gw / gb (the critics' weights only carry it to their action inputs).
 * The critic pass reads actor, critic, critic2 and both target critics; the actor pass reads
 * actor, critic and critic2. */
typedef struct wdb_tqc_update_args {
  int n_envs, n_agents, obs_dim, action_dim;   /* E, Np, F, A (the actor's head is 2A wide) */
  int capacity, n_step;              /* ring slots C, n-step horizon (n_step + 1 <= C) */
  int n_quantiles, n_drop;           /* N per critic, the top quantiles dropped per critic */
  float gamma, action_scale, action_bias;
  float log_std_min, log_std_max;
  const float *log_alpha;            /* device [1] */
  const float *obs;                  /* [C, E, Np, F] */
  const float *actions;              /* [C, E, Np, A] */
  const float *rewards;              /* [C, E, Np] */
  const int *done;                   /* [C, E] */
  const float *critic_noise;         /* [B, A] standard normal (eps') */
  const float *actor_noise;          /* [B, A] (eps) */
  wdb_ddpg_net actor, critic, critic2;          /* gradients: actor (actor pass), critics */
  wdb_ddpg_net target_critic, target_critic2;   /* the critic's shape, head N */
  float *q_means, *target_means;     /* critic pass out [B]: mean_m,i theta, mean_k T_k; or NULL */
  float *log_probs;                  /* actor pass out [B]: log pi(a | obs), or NULL */
  double *sums;                      /* out [4]: sum_g loss_g, sum_g mean theta (critic pass),
                                        sum_g Qbar_g, sum_g log pi (actor pass) */
  void *workspace;                   /* the pass's _workspace_bytes() bytes */
} wdb_tqc_update_args;
/* 1 if a pass takes the shapes: 0..3 hidden layers of width 1..64 per network, the four critics
 * shaped alike, 2 <= N and 2N <= 64, 0 <= n_drop < N, A <= 32, F + A <= 64, E, Np >= 1,
 * 1 <= n_step, n_step + 1 <= capacity, n_windows >= 1, log_std_min <= log_std_max, and the pass's
 * networks, gradient blocks and row tiles in one CTA's shared memory (the critic pass holds the
 * actor, four critics, two gradient blocks and 8 + 2 (hidden layers) row tiles).  No CUDA call. */
int wdb_tqc_critic_update_sampled_supported(const wdb_tqc_update_args *update, int n_windows);
long long wdb_tqc_critic_update_sampled_workspace_bytes(const wdb_tqc_update_args *update,
                                                        int n_windows);   /* -1: unsupported */
int wdb_tqc_actor_update_sampled_supported(const wdb_tqc_update_args *update, int n_windows);
long long wdb_tqc_actor_update_sampled_workspace_bytes(const wdb_tqc_update_args *update,
                                                       int n_windows);    /* -1: unsupported */
/* cudaErrorInvalidValue without launching if unsupported or a required pointer is NULL. */
int wdb_tqc_critic_update_sampled(void *stream, const wdb_tqc_update_args *update,
                                  const wdb_replay_windows *windows);
int wdb_tqc_actor_update_sampled(void *stream, const wdb_tqc_update_args *update,
                                 const wdb_replay_windows *windows);

/* ---- recurrent policies (csrc/wdb_recurrent.cu) ----------------------------------------------
 * FullyConnectedGRU's per-step rollout forward: n_layers (0..2) Linear + ReLU trunk layers, an
 * nn.GRUCell of width H (gate order r, z, n) and one softmax head per discrete action head,
 * reading the new state h' (head_kind 0), or FullyConnectedGaussianGRU's one raw mean head
 * (head_kind 1).  fp32 throughout; the value head is not evaluated.  Weights are the torch
 * parameters as they are (Linear [out, in], weight_ih [3H, D], weight_hh [3H, H]). */
typedef struct wdb_gru_forward {
  long long n_rows;                  /* R = E * Np */
  int in_dim;                        /* F */
  int n_layers;                      /* trunk layers, 0 .. 2 */
  int dims[2];                       /* their widths (dims[l] for l < n_layers) */
  int hidden_size;                   /* H */
  int n_heads;                       /* 1 or 2 */
  int heads[2];                      /* A_k for k < n_heads */
  const float *obs;                  /* [R, F] */
  float *hidden;                     /* [R, H]: h in, h' out (in place) */
  const float *fc_weight[2], *fc_bias[2];
  const float *weight_ih, *weight_hh, *bias_ih, *bias_hh;
  const float *head_weight[2], *head_bias[2];
  float *probs[2];                   /* out [R, A_k] */
  int head_kind;                     /* 0: softmax heads (probs[k] = the head's probabilities);
                                        1: one raw mean head, n_heads == 1: probs[0] = the mean
                                        [R, A], A = heads[0] (no softmax, no tanh) */
} wdb_gru_forward;
/* Dynamic shared memory of wdb_gru_policy_forward at these shapes; 0 if it refuses them:
 * 1 <= F <= 256, trunk widths and H in 1 .. 128, 1 or 2 heads of 1 .. 64 actions, and the
 * weights plus a 16-row tile of activations in 227 KB.  A mean head of A dimensions is asked
 * as one head of A actions (n_heads 1, a0 = A); both kinds take the same bytes.  No CUDA call. */
long long wdb_gru_forward_bytes(int in_dim, int n_layers, int d0, int d1, int hidden_size,
                                int n_heads, int a0, int a1);
/* One launch: h' into `hidden`, the heads' probabilities (or the mean) into probs[k].  Each
 * output is one thread's k-ascending fmaf sum plus its bias; sig(x) = 1 / (1 + expf(-x)),
 * tanh = tanhf.  h' does not depend on head_kind.  Bit-identical on relaunch.
 * cudaErrorInvalidValue without launching on refused shapes, a NULL pointer, an unknown
 * head_kind or head_kind 1 with n_heads != 1. */
int wdb_gru_policy_forward(void *stream, const wdb_gru_forward *args);

#define WDB_RECURRENT_MAX_POLICIES 8
typedef struct wdb_recurrent_state {
  float *hidden;                     /* [E, Np, H] */
  int n_agents;                      /* Np */
  int hidden_size;                   /* H */
} wdb_recurrent_state;
typedef struct wdb_recurrent_reset {
  const int *done;                   /* [E] the env's _done_ */
  int n_envs;
  int n_policies;                    /* 1 .. WDB_RECURRENT_MAX_POLICIES */
  wdb_recurrent_state policy[WDB_RECURRENT_MAX_POLICIES];
} wdb_recurrent_reset;
/* Zeroes hidden[e, :, :] of every listed policy for every env e with done[e] > 0, one launch. */
int wdb_recurrent_reset_done(void *stream, const wdb_recurrent_reset *table);

#ifdef __cplusplus
}
#endif
#endif /* WDB200_H_ */
