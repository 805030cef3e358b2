// wdb_sa_rollout.cu -- the WHOLE T-step rollout of a single-agent classic-control env in ONE
// launch: policy forward -> action sample -> env.step -> reward / done bookkeeping ->
// done-masked reset -> push to the training batch, T times; eight lanes share one env replica
// (the forward pass is split over them, lane 0 does the serial part of the timestep).
// Discrete kinds (CartPole, MountainCar, Acrobot; BASELINE config 3: CartPole x 10 000
// replicas) sample a softmax head; continuous kinds (ContinuousMountainCar, Pendulum: the
// DDPG configs) evaluate the actor's tanh head and add Ornstein-Uhlenbeck exploration noise.
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
#include <type_traits>

#include "wdb_sa_physics.cuh"

using namespace wdb;

namespace {

constexpr int kSaThreads = 64;
constexpr int kSaGroup = 8;         // lanes that share one env replica's forward pass
constexpr int kSaEnvsPerCta = kSaThreads / kSaGroup;
constexpr int kSaMaxWidth = 64;     // widest layer (and observation) held per env
constexpr int kSaPitch = kSaMaxWidth + 1;  // activation row pitch (odd: no bank conflicts)
constexpr int kSaMaxWeights = 11 * 1024;   // floats of shared memory for the policy

__device__ __forceinline__ int sa_search(const float *cdf, float p, int r) {
  int left = 0, right = r;                     // search_index, core/random.cu:33-49
  while (left <= right) {
    const int mid = left + (right - left) / 2;
    const float v = cdf[mid];
    if (fabsf(v - p) < 1.0e-8f) return mid;
    if (v < p) left = mid + 1; else right = mid - 1;
  }
  return left > r ? r : left;
}

// Thread layout: kSaGroup = 8 consecutive lanes own one env replica.  The forward pass is
// split over the group (lane `sub` computes output neurons sub, sub + 8, ... of every layer;
// each neuron still accumulates bias + w[0] x[0] + w[1] x[1] + ... in that order, so the
// result does not depend on the split); activations travel through a per-env shared-memory
// row, the weights sit TRANSPOSED in shared memory (Wt[i][j]: the lanes of a group read
// consecutive words, the groups of a warp the same words).  Lane 0 of the group then does the
// serial part of the timestep -- softmax, sample, physics, bookkeeping, reset -- so the
// dependent chain per timestep is ~1/7 of a one-thread-per-env layout and eight times as many
// warps are in flight.  All control flow is warp-uniform (groups past n_envs compute on
// clamped indices and skip their stores).
// Residency: the kernel loops over ALL timesteps, so a grid that does not fit the GPU in ONE
// wave pays the whole rollout twice.  At 128 registers 8 CTAs of 64 threads fit an SM: 1056
// slots on 132 SMs for BASELINE config 3's 1250 CTAs (10 000 envs) -- 1.18 waves, the last
// envs would double the time.  Capped at 96 registers 10 CTAs fit: 1320 slots.
// (16-byte weight / activation loads in the forward, 5 loads per 16 FMAs instead of 20, do
// not help: the step is bound by lane 0's serial softmax / sample / physics chain, not by
// the forward's load count.)
// kContinuous: Pendulum / ContinuousMountainCar (deterministic tanh head + OU exploration,
// float32 actions) instead of the softmax head + categorical sample; a compile-time switch,
// so the discrete instantiation is the code it was before the continuous kinds existed.
template <bool kContinuous>
__global__ void __launch_bounds__(kSaThreads, 9)
sa_rollout_kernel(const __grid_constant__ wdb_sa_rollout R) {
  extern __shared__ float s_w[];               // per layer: [Wt (in x out) | b (out)]
  __shared__ int s_dims[8];                    // layer widths (dynamic indexing of the kernel
  if (threadIdx.x < 5) s_dims[threadIdx.x] = R.dims[threadIdx.x];   // parameter goes through
  __syncthreads();                             // local memory: do it once)
  const int n_layers = R.n_hidden + 1;
  int w_floats = 0;
  for (int l = 0; l < n_layers; l++) {
    const int in = s_dims[l], out = s_dims[l + 1];
    for (int i = threadIdx.x; i < in * out; i += blockDim.x) {
      const int j = i / in, k = i - j * in;    // W[j][k] (nn.Linear: [out, in]) -> Wt[k][j]
      s_w[w_floats + k * out + j] = R.w[l][i];
    }
    for (int i = threadIdx.x; i < out; i += blockDim.x) s_w[w_floats + in * out + i] = R.b[l][i];
    w_floats += in * out + out;
  }
  float *s_act = s_w + w_floats;               // [kSaEnvsPerCta][2][kSaPitch]
  __syncthreads();
  const int sub = threadIdx.x & (kSaGroup - 1);
  const int env_local = threadIdx.x / kSaGroup;
  const int env_raw = blockIdx.x * kSaEnvsPerCta + env_local;
  const bool live = env_raw < R.n_envs;
  const int env = live ? env_raw : R.n_envs - 1;
  const bool lead = live && sub == 0;
  const int E = R.n_envs, F = s_dims[0], A = s_dims[n_layers];
  float *buf0 = s_act + (env_local * 2 + 0) * kSaPitch;
  float *buf1 = s_act + (env_local * 2 + 1) * kSaPitch;

  RngHeader rh = {0ull, 0ull}, ph = {0ull, 0ull};
  unsigned long long rng_off = 0, pool_off = 0;
  float run = 0.0f, ou = 0.0f;
  int steps_run = 0, tstep = 0, done_flag = 0;
  if (lead) {
    if (R.rng_state) {
      rh = *reinterpret_cast<const RngHeader *>(R.rng_state);
      rng_off = rng_offsets(R.rng_state)[env];
    }
    if (R.pool_rng) {
      ph = *reinterpret_cast<const RngHeader *>(R.pool_rng);
      pool_off = rng_offsets(R.pool_rng)[env];
    }
    run = R.reward_running_sum ? R.reward_running_sum[env] : 0.0f;
    steps_run = R.step_running_sum ? R.step_running_sum[env] : 0;
    tstep = R.env_timestep[env];
    done_flag = R.done[env];
    if constexpr (kContinuous) {
      if (R.ou_state) ou = R.ou_state[env];
    }
  }

  for (int t = 0; t < R.n_steps; t++) {
    // ---- observation -> activation row 0 and batch slot t (model_base.py:181-200)
    {
      const float *obs = R.observations + (size_t)env * F;
      float *ob = R.obs_batch ? R.obs_batch + ((size_t)t * E + env) * F : nullptr;
      for (int i = sub; i < F; i += kSaGroup) {
        const float x = obs[i];
        buf0[i] = x;
        if (ob && live) ob[i] = x;
      }
    }
    __syncwarp();
    // ---- policy forward (fully_connected.py:51-89): Linear + ReLU hidden layers, linear head
    float *cur = buf0, *nxt = buf1;
    int off = 0;
    for (int l = 0; l < n_layers; l++) {
      const int in = s_dims[l], out = s_dims[l + 1];
      const float *Wt = s_w + off, *bl = Wt + in * out;
      // this lane's output neurons sub, sub + 8, ... in blocks of four that accumulate side
      // by side: one broadcast load of x[i] feeds four independent FMA chains (each neuron
      // still sums bias, w[0] x[0], w[1] x[1], ... in that order)
      for (int jb = sub; jb < out; jb += 4 * kSaGroup) {
        const int last = out - 1;                       // clamp: lanes past `out` re-read a valid word
        const int j0 = jb, j1 = min(jb + kSaGroup, last), j2 = min(jb + 2 * kSaGroup, last),
                  j3 = min(jb + 3 * kSaGroup, last);
        float a0 = bl[j0], a1 = bl[j1], a2 = bl[j2], a3 = bl[j3];
        const float *wr = Wt;
        for (int i = 0; i < in; i++, wr += out) {
          const float x = cur[i];
          a0 = fmaf(wr[j0], x, a0);
          a1 = fmaf(wr[j1], x, a1);
          a2 = fmaf(wr[j2], x, a2);
          a3 = fmaf(wr[j3], x, a3);
        }
        const bool hidden = l < n_layers - 1;
        nxt[j0] = hidden ? fmaxf(a0, 0.0f) : a0;
        if (jb + kSaGroup < out) nxt[jb + kSaGroup] = hidden ? fmaxf(a1, 0.0f) : a1;
        if (jb + 2 * kSaGroup < out) nxt[jb + 2 * kSaGroup] = hidden ? fmaxf(a2, 0.0f) : a2;
        if (jb + 3 * kSaGroup < out) nxt[jb + 3 * kSaGroup] = hidden ? fmaxf(a3, 0.0f) : a3;
      }
      off += in * out + out;
      __syncwarp();
      float *tmp = cur; cur = nxt; nxt = tmp;
    }
    if (lead) {
      std::conditional_t<kContinuous, float, int> action;
      if constexpr (kContinuous) {
        // deterministic head (FullyConnectedActor._policy_outputs): scale * tanh(z) + bias,
        // a separate multiply and add as torch evaluates it
        const float mean = __fadd_rn(__fmul_rn(R.action_scale, tanhf(cur[0])), R.action_bias);
        if (R.probs_batch) R.probs_batch[(size_t)t * E + env] = mean;
        // ---- OU exploration (sample_ou_process): the stand-alone sampler's own update
        const OuStep o = ou_step(mean, ou, R.normals ? R.normals + (size_t)t * E + env : nullptr,
                                 rh, (unsigned long long)env, rng_off, R.ou_damping,
                                 R.ou_stddev, R.ou_scale);
        ou = o.ou;
        rng_off += o.draws;
        action = o.action;
        static_cast<float *>(R.sampled_actions)[env] = action;
        if (R.actions_batch) static_cast<float *>(R.actions_batch)[(size_t)t * E + env] = action;
      } else {
        // softmax over the A logits in cur[] (torch.softmax: subtract the max, exp, normalise)
        float mx = cur[0];
        for (int i = 1; i < A; i++) mx = fmaxf(mx, cur[i]);
        float z = 0.0f;
        for (int i = 0; i < A; i++) { cur[i] = expf(cur[i] - mx); z += cur[i]; }
        for (int i = 0; i < A; i++) cur[i] = cur[i] / z;
        if (R.probs_batch) {
          float *pb = R.probs_batch + ((size_t)t * E + env) * A;
          for (int i = 0; i < A; i++) pb[i] = cur[i];
        }
        // ---- categorical sample (core/random.cu:51-85): u in (0, 1], float32 CDF, binary search
        float u;
        if (R.uniforms) {
          u = R.uniforms[(size_t)t * E + env];
        } else {
          u = u32_to_uniform(rng_draw4(rh, (unsigned long long)env, rng_off).x);
          rng_off++;
        }
        if (R.use_argmax) {
          action = 0;
          float best = cur[0];
          for (int i = 1; i < A; i++) if (best < cur[i]) { best = cur[i]; action = i; }
        } else {
          float c = cur[0];
          for (int i = 1; i < A; i++) { c = cur[i] + c; cur[i] = c; }
          action = sa_search(cur, u, A - 1);
        }
        static_cast<int *>(R.sampled_actions)[env] = action;
        if (R.actions_batch) static_cast<int *>(R.actions_batch)[(size_t)t * E + env] = action;
      }

      // ---- env step: the stand-alone step kernel's own step function
      tstep += 1;
      float *st = R.state, *ob = R.observations;
      const float *p = R.env_params;
      const int T = R.episode_length;
      SaStepOut s;
      if constexpr (kContinuous) {
        if (R.env_kind == WDB_SA_CONTINUOUS_MOUNTAIN_CAR)
          s = sa_env_step<WDB_SA_CONTINUOUS_MOUNTAIN_CAR>(st, ob, env, action, p, tstep, T);
        else
          s = sa_env_step<WDB_SA_PENDULUM>(st, ob, env, action, p, tstep, T);
      } else {
        if (R.env_kind == WDB_SA_CARTPOLE)
          s = sa_env_step<WDB_SA_CARTPOLE>(st, ob, env, action, p, tstep, T);
        else if (R.env_kind == WDB_SA_MOUNTAIN_CAR)
          s = sa_env_step<WDB_SA_MOUNTAIN_CAR>(st, ob, env, action, p, tstep, T);
        else
          s = sa_env_step<WDB_SA_ACROBOT>(st, ob, env, action, p, tstep, T);
      }
      const float reward = s.reward;
      R.rewards[env] = reward;
      // the reference's done flag is sticky until a reset clears it
      if (s.done) done_flag = s.done;

      // ---- bookkeeping (trainer_base.py:514-601): batch slots, running episodic sums
      if (R.rewards_batch) R.rewards_batch[(size_t)t * E + env] = reward;
      if (R.done_batch) R.done_batch[(size_t)t * E + env] = done_flag;
      run += reward;
      steps_run += 1;
      if (done_flag > 0) {
        if (R.episodic_reward_sum) atomicAdd(R.episodic_reward_sum, run);
        if (R.episodic_step_sum) atomicAdd(R.episodic_step_sum, (unsigned long long)steps_run);
        if (R.num_completed) atomicAdd(R.num_completed, 1ull);
        run = 0.0f;
        steps_run = 0;
      }

      // ---- done-masked reset (core/reset.cu:9-75, pool_reset.py:15-52)
      if (done_flag > 0 && R.reset_done_envs) {
        int n_pool = 0;
        for (int arr = 0; arr < R.n_reset_arrays; arr++) {
          const wdb_reset_desc d = R.reset_table[arr];
          const long long words = d.bytes_per_env >> 2;
          const long long src_row = reset_src_row(d, ph, env, pool_off, n_pool);
          uint32_t *dst = reinterpret_cast<uint32_t *>(
              reinterpret_cast<char *>(d.dst) + (long long)env * d.bytes_per_env);
          const uint32_t *src = reinterpret_cast<const uint32_t *>(
              reinterpret_cast<const char *>(d.ref) + src_row * d.bytes_per_env);
          for (long long i = 0; i < words; i++) dst[i] = src[i];
        }
        pool_off += n_pool;
        done_flag = 0;
        tstep = 0;
      }
    }
    // the group's other lanes read the observation row lane 0 just wrote (global memory)
    __threadfence_block();
    __syncwarp();
  }
  if (lead) {
    R.env_timestep[env] = tstep;
    R.done[env] = done_flag;
    if constexpr (kContinuous) {
      if (R.rng_state && !R.normals) rng_offsets(R.rng_state)[env] = rng_off;
      if (R.ou_state) R.ou_state[env] = ou;
    } else {
      if (R.rng_state && !R.uniforms) rng_offsets(R.rng_state)[env] = rng_off;
    }
    if (R.pool_rng) rng_offsets(R.pool_rng)[env] = pool_off;
    if (R.reward_running_sum) R.reward_running_sum[env] = run;
    if (R.step_running_sum) R.step_running_sum[env] = steps_run;
  }
}

}  // namespace

WDB_API int wdb_single_agent_rollout_supported(int n_hidden, const int *dims) {
  if (n_hidden < 0 || n_hidden > 3 || !dims) return 0;
  long long total = 0;
  for (int l = 0; l <= n_hidden + 1; l++)
    if (dims[l] < 1 || dims[l] > kSaMaxWidth) return 0;
  for (int l = 0; l <= n_hidden; l++) total += (long long)dims[l] * dims[l + 1] + dims[l + 1];
  return total <= kSaMaxWeights ? 1 : 0;
}

namespace {
template <bool kContinuous>
int sa_launch(void *stream, const wdb_sa_rollout *r, size_t smem) {
  static size_t configured = 0;
  if (smem > 48 * 1024 && smem > configured) {
    cudaError_t e = cudaFuncSetAttribute(sa_rollout_kernel<kContinuous>,
                                         cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return (int)e;
    configured = smem;
  }
  const int grid = (r->n_envs + kSaEnvsPerCta - 1) / kSaEnvsPerCta;
  sa_rollout_kernel<kContinuous><<<grid, kSaThreads, smem, as_stream(stream)>>>(*r);
  return finish_launch();
}
}  // namespace

WDB_API int wdb_single_agent_rollout(void *stream, const wdb_sa_rollout *r) {
  if (!r) return (int)cudaErrorInvalidValue;
  const int rc = sa_check_env_arrays(r->env_kind, r->n_envs, r->state, r->sampled_actions,
                                     r->done, r->rewards, r->observations, r->env_timestep);
  if (rc != cudaSuccess) return rc;
  const bool continuous = r->env_kind >= WDB_SA_CONTINUOUS_MOUNTAIN_CAR;
  if (r->n_steps <= 0) return (int)cudaErrorInvalidValue;
  if (!wdb_single_agent_rollout_supported(r->n_hidden, r->dims)) return (int)cudaErrorInvalidValue;
  for (int l = 0; l <= r->n_hidden; l++)
    if (!r->w[l] || !r->b[l]) return (int)cudaErrorInvalidValue;
  if (continuous) {
    // the OU state and a normal source unless the bypass (scale < 1e-8) draws nothing
    if (!(r->ou_scale < 1.0e-8f) && (!r->ou_state || (!r->normals && !r->rng_state)))
      return (int)cudaErrorInvalidValue;
  } else if (!r->use_argmax && !r->uniforms && !r->rng_state) {
    return (int)cudaErrorInvalidValue;
  }
  // the observation feeds the first layer, and the head is one logit per discrete action
  // (one tanh output for the continuous kinds): a wider head would step the env with actions
  // it does not have
  if (r->state_dim != kSaStateDim[r->env_kind] || r->dims[0] != kSaObsDim[r->env_kind] ||
      r->dims[r->n_hidden + 1] != kSaNActions[r->env_kind])
    return (int)cudaErrorInvalidValue;
  if (r->reset_done_envs && r->n_reset_arrays > 0 && !r->reset_table)
    return (int)cudaErrorInvalidValue;
  long long total = 0;
  for (int l = 0; l <= r->n_hidden; l++)
    total += (long long)r->dims[l] * r->dims[l + 1] + r->dims[l + 1];
  const size_t smem = ((size_t)total + (size_t)kSaEnvsPerCta * 2 * kSaPitch) * sizeof(float);
  return continuous ? sa_launch<true>(stream, r, smem) : sa_launch<false>(stream, r, smem);
}
