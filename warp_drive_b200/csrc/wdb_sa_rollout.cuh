// wdb_sa_rollout.cuh -- the one-launch single-agent rollout kernel (see wdb_sa_rollout.cu for
// what it does and why) and its launcher, one template over the action head.  wdb_sa_rollout.cu
// instantiates the softmax, tanh / OU, Gaussian, squashed Gaussian and Q heads;
// wdb_sa_rollout_categorical.cu the categorical Q head, wdb_sa_rollout_noisy.cu the noisy Q head
// and wdb_sa_rollout_obs_norm.cu the softmax and Gaussian heads on normalized observations, each
// in a translation unit of its own so that the other kinds keep their file and machine code.  Each translation unit gets its own
// copy (anonymous namespace).
#pragma once

#include <type_traits>

#include "wdb_noisy.cuh"
#include "wdb_obs_norm.cuh"
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

// The categorical head's expectation of one block of N atom logits y over a group's lanes
// (lane sub: atoms sub, sub + 8, ... in order, then an xor butterfly over the 8 lanes):
// sum_j z_j e_j / sum_j e_j, e_j = expf(y_j - max y).  Every lane returns the same bits.
static __device__ __noinline__ float sa_expectation(const float *y, const float *z, int N,
                                                    int sub) {
  float mx = -INFINITY;
  for (int j = sub; j < N; j += kSaGroup) mx = fmaxf(mx, y[j]);
  for (int o = kSaGroup / 2; o > 0; o /= 2)
    mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o, kSaGroup));
  float s = 0.0f, q = 0.0f;
  for (int j = sub; j < N; j += kSaGroup) {
    const float e = expf(y[j] - mx);
    s += e;
    q = fmaf(z[j], e, q);
  }
  for (int o = kSaGroup / 2; o > 0; o /= 2) {
    s += __shfl_xor_sync(0xffffffffu, s, o, kSaGroup);
    q += __shfl_xor_sync(0xffffffffu, q, o, kSaGroup);
  }
  return __fdiv_rn(q, s);
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
// kKind: the action head, a compile-time switch, so each instantiation is the code it was
// before the later heads existed.  kSaSoftmax: softmax head + categorical sample (int32
// actions); kSaTanhOu: Pendulum / ContinuousMountainCar with a deterministic tanh head + OU
// exploration; kSaGaussian: the same envs with a Gaussian head (raw linear mean, log_std) and
// gaussian_step; kSaSquashed: the same envs with SAC's squashed Gaussian head (2 wide: mu, raw
// log-std) and squashed_gaussian_step -- float32 actions for all three.  kSaEpsGreedy: the
// discrete kinds with DQN's Q head (raw outputs) and epsilon_greedy_step (int32 actions).
// kSaCategoricalQ: the discrete kinds with C51's categorical head -- A blocks of N atom logits,
// each reduced to its expectation over the group's lanes -- and epsilon_greedy_step on those.
// kSaNoisyQ: the discrete kinds with a noisy DQN head (one NoisyLinear, A <= 3 outputs): output
// j is fmaf(f(eps_out)_j, sigma_b_j + sum_i sigma_W[j][i] (f(eps_in)_i h_i), mu-part_j), the
// mu-part computed exactly as the Q kind's head, fresh noise (noisy_f) per env row and step;
// use_argmax: the mu-part alone.  Then epsilon_greedy_step.
// kSaSoftmaxNorm, kSaGaussianNorm: the softmax and Gaussian kinds with the observation
// normalized (obs_normalize) as it enters activation row 0; the batch slot keeps the raw x.
// [shift F | scale F | clip] sit in the device buffer behind log_std (after the Gaussian
// head's log-std).  (Each test of the kind is an `if constexpr` or a constant that the earlier
// kinds evaluate as before: their machine code is unchanged.)
// noisy_f as a call: the noisy kind's Philox, logf and cosf stay out of the rollout loop's
// registers (inlined, they push the kernel past its register budget into spills)
__device__ __noinline__ float sa_noise(unsigned long long seed, unsigned long long step,
                                       uint32_t env, int e) {
  return noisy_f(seed, 1, step, env, 0, e);
}

enum { kSaSoftmax = 0, kSaTanhOu = 1, kSaGaussian = 2, kSaSquashed = 3, kSaEpsGreedy = 4,
       kSaCategoricalQ = 5, kSaNoisyQ = 6, kSaSoftmaxNorm = 7, kSaGaussianNorm = 8 };
template <int kKind>
__global__ void __launch_bounds__(kSaThreads, 9)
sa_rollout_kernel(const __grid_constant__ wdb_sa_rollout R) {
  constexpr bool kContinuous = kKind != kSaSoftmax && kKind != kSaEpsGreedy &&
                               kKind != kSaCategoricalQ && kKind != kSaNoisyQ &&
                               kKind != kSaSoftmaxNorm;
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
  // categorical head: the discrete kind's action count, each env's Q row ([kSaEnvsPerCta]
  // [kSaPitch] after the activation rows), then the support (log_std[1 ..])
  // (s_dims[5], s_dims[6] = the action count and N)
  if constexpr (kKind == kSaCategoricalQ) {
    const int n_q = R.env_kind == WDB_SA_CARTPOLE ? 2 : 3, n_atoms = R.dims[n_layers] / n_q;
    float *s_z = s_act + kSaEnvsPerCta * 3 * kSaPitch;
    for (int i = threadIdx.x; i < n_atoms; i += blockDim.x) s_z[i] = R.log_std[1 + i];
    if (threadIdx.x == 0) {
      s_dims[5] = n_q;
      s_dims[6] = n_atoms;
    }
  }
  // noisy head: sigma_W [A][H] and sigma_b [A] after the activation rows (log_std[5 ..])
  if constexpr (kKind == kSaNoisyQ) {
    const int n_sigma = R.dims[n_layers] * R.dims[n_layers - 1] + R.dims[n_layers];
    float *s_sig = s_act + kSaEnvsPerCta * 2 * kSaPitch;
    for (int i = threadIdx.x; i < n_sigma; i += blockDim.x) s_sig[i] = R.log_std[5 + i];
  }
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
  float run = 0.0f, ou = 0.0f, ls_lo = 0.0f, ls_hi = 0.0f, eps = 0.0f;
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
    if constexpr (kKind == kSaTanhOu) {
      if (R.ou_state) ou = R.ou_state[env];
    }
    if constexpr (kKind == kSaSquashed) {
      ls_lo = R.log_std[0];
      ls_hi = R.log_std[1];
    }
    if constexpr (kKind == kSaEpsGreedy || kKind == kSaCategoricalQ || kKind == kSaNoisyQ)
      eps = R.use_argmax ? 0.0f : R.log_std[0];
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
      // the normalizing kinds: each lane normalizes the elements it just wrote
      if constexpr (kKind == kSaSoftmaxNorm || kKind == kSaGaussianNorm) {
        const float *nrm = R.log_std + (kKind == kSaGaussianNorm ? 1 : 0);
        for (int i = sub; i < F; i += kSaGroup)
          buf0[i] = obs_normalize(buf0[i], nrm[i], nrm[F + i], nrm[2 * F]);
      }
    }
    __syncwarp();
    // ---- policy forward (fully_connected.py:51-89): Linear + ReLU hidden layers, linear head
    float *cur = buf0, *nxt = buf1;
    int off = 0;
    // (the categorical head runs after the loop, block by block)
    // (so does the noisy head)
    const int n_fwd = kKind == kSaCategoricalQ || kKind == kSaNoisyQ ? n_layers - 1 : n_layers;
    for (int l = 0; l < n_fwd; l++) {
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
    if constexpr (kKind == kSaCategoricalQ) {
      // the head as n_q blocks of N atom logits: block a (head rows a N .. a N + N - 1) into
      // the activation row, split over the lanes as the layers above; then Q[a] over the
      // group's lanes (sa_expectation) into the env's Q row
      const int n_q = s_dims[5], N = s_dims[6];
      const int in = s_dims[n_layers - 1], out = s_dims[n_layers];
      const float *Wt = s_w + off, *bl = Wt + in * out;
      const float *s_z = s_act + kSaEnvsPerCta * 3 * kSaPitch;
      float *qrow = s_act + (kSaEnvsPerCta * 2 + env_local) * kSaPitch;
      for (int a = 0; a < n_q; a++) {
        const int c0 = a * N;
        for (int jb = sub; jb < N; jb += 2 * kSaGroup) {   // two side by side (registers)
          const int j0 = jb, j1 = min(jb + kSaGroup, N - 1);
          float a0 = bl[c0 + j0], a1 = bl[c0 + j1];
          const float *wr = Wt + c0;
          for (int i = 0; i < in; i++, wr += out) {
            const float x = cur[i];
            a0 = fmaf(wr[j0], x, a0);
            a1 = fmaf(wr[j1], x, a1);
          }
          nxt[j0] = a0;
          if (jb + kSaGroup < N) nxt[jb + kSaGroup] = a1;
        }
        __syncwarp();
        const float qa = sa_expectation(nxt, s_z, N, sub);
        if (sub == 0) qrow[a] = qa;
        __syncwarp();
      }
      cur = qrow;
    }
    if constexpr (kKind == kSaNoisyQ) {
      // f(eps_in) * h into the spare activation row (lanes split i as the layers above), then
      // lane j < A computes output j: the Q kind's mu-part, then the sigma part and f(eps_out)_j
      const int in = s_dims[n_layers - 1], out = s_dims[n_layers];
      const float *Wt = s_w + off, *bl = Wt + in * out;
      const float *sw = s_act + kSaEnvsPerCta * 2 * kSaPitch, *sb = sw + out * in;
      const bool noisy = !R.use_argmax;
      // the noise key: log_std[1 .. 4] as raw words (seed, then the acting step of t = 0), read
      // here rather than held across the loop (registers)
      const uint32_t *kw = reinterpret_cast<const uint32_t *>(R.log_std) + 1;
      const unsigned long long noise_seed =
          (unsigned long long)kw[0] | ((unsigned long long)kw[1] << 32);
      const unsigned long long step =
          ((unsigned long long)kw[2] | ((unsigned long long)kw[3] << 32)) + (unsigned long long)t;
      if (noisy) {
        for (int i = sub; i < in; i += kSaGroup)
          nxt[i] = sa_noise(noise_seed, step, (uint32_t)env, i) * cur[i];
        __syncwarp();
      }
      float q = 0.0f;
      if (sub < out) {
        float a = bl[sub];
        const float *wr = Wt;
        for (int i = 0; i < in; i++, wr += out) a = fmaf(wr[sub], cur[i], a);
        if (noisy) {
          float sg = sb[sub];
          for (int i = 0; i < in; i++) sg = fmaf(sw[sub * in + i], nxt[i], sg);
          a = fmaf(sa_noise(noise_seed, step, (uint32_t)env, in + sub), sg, a);
        }
        q = a;
      }
      __syncwarp();                                     // every lane has read h
      if (sub < out) cur[sub] = q;
      __syncwarp();
    }
    if (lead) {
      std::conditional_t<kContinuous, float, int> action;
      if constexpr (kKind == kSaSquashed) {
        // squashed Gaussian head: the stand-alone sampler's own step on [mu, raw log-std]
        if (R.probs_batch) R.probs_batch[(size_t)t * E + env] = cur[0];
        float *dst = static_cast<float *>(R.sampled_actions) + env;
        rng_off += squashed_gaussian_step(
            cur, dst, 1, R.action_scale, R.action_bias, ls_lo, ls_hi,
            R.normals ? R.normals + (size_t)t * E + env : nullptr, rh, (unsigned long long)env,
            rng_off, R.use_argmax);
        action = *dst;
        if (R.actions_batch) static_cast<float *>(R.actions_batch)[(size_t)t * E + env] = action;
      } else if constexpr (kKind == kSaGaussian || kKind == kSaGaussianNorm) {
        // Gaussian head: the raw linear output is the mean; the stand-alone sampler's own step
        // writes the action straight into sampled_actions
        if (R.probs_batch) R.probs_batch[(size_t)t * E + env] = cur[0];
        float *dst = static_cast<float *>(R.sampled_actions) + env;
        rng_off += gaussian_step(cur, R.log_std, dst, 1,
                                 R.normals ? R.normals + (size_t)t * E + env : nullptr, rh,
                                 (unsigned long long)env, rng_off, R.use_argmax);
        action = *dst;
        if (R.actions_batch) static_cast<float *>(R.actions_batch)[(size_t)t * E + env] = action;
      } else if constexpr (kContinuous) {
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
      } else if constexpr (kKind == kSaEpsGreedy || kKind == kSaCategoricalQ ||
                           kKind == kSaNoisyQ) {
        // Q head: the raw outputs are the Q values (categorical head: the expectations); the
        // stand-alone sampler's own rule, one draw of stream `env` per step (epsilon read once
        // above; use_argmax: 0, greedy)
        const int nA = kKind == kSaCategoricalQ ? s_dims[5] : A;
        if (R.probs_batch) {
          float *pb = R.probs_batch + ((size_t)t * E + env) * nA;
          for (int i = 0; i < nA; i++) pb[i] = cur[i];
        }
        action = epsilon_greedy_step(cur, nA, eps, nullptr, rh, (unsigned long long)env,
                                     rng_off);
        rng_off++;
        static_cast<int *>(R.sampled_actions)[env] = action;
        if (R.actions_batch) static_cast<int *>(R.actions_batch)[(size_t)t * E + env] = action;
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
      if constexpr (kKind == kSaTanhOu) {
        if (R.ou_state) R.ou_state[env] = ou;
      }
    } else {
      if (R.rng_state && !R.uniforms) rng_offsets(R.rng_state)[env] = rng_off;
    }
    if (R.pool_rng) rng_offsets(R.pool_rng)[env] = pool_off;
    if (R.reward_running_sum) R.reward_running_sum[env] = run;
    if (R.step_running_sum) R.step_running_sum[env] = steps_run;
  }
}

template <int kKind>
int sa_launch(void *stream, const wdb_sa_rollout *r, size_t smem) {
  static size_t configured = 0;
  if (smem > 48 * 1024 && smem > configured) {
    cudaError_t e = cudaFuncSetAttribute(sa_rollout_kernel<kKind>,
                                         cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return (int)e;
    configured = smem;
  }
  const int grid = (r->n_envs + kSaEnvsPerCta - 1) / kSaEnvsPerCta;
  sa_rollout_kernel<kKind><<<grid, kSaThreads, smem, as_stream(stream)>>>(*r);
  return finish_launch();
}

}  // namespace
