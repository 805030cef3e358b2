// wdb_update.cu -- the fused pieces of the A2C / PPO update (SURVEY.md section 8 row f1).
//
// (1) pg_loss_kernel: ONE backward-in-time scan per (env, agent) over the [T, E, Np] batch that
//     produces everything between the policy forward and the backward pass of the reference's
//     update (warp_drive/training/algorithms/policygradient/a2c.py:80-130, ppo.py:82-141):
//     bootstrapped discounted returns with done masking, advantages, the Categorical log-prob
//     of the taken action and the entropy of every action head, the three loss sums (policy,
//     value, entropy) AND the gradients of the total loss with respect to the probabilities
//     and the values.  The reference builds the same quantities out of ~40 elementwise torch
//     kernels per head plus ~6 per timestep for the returns recursion, and autograd then walks
//     that graph backwards.
// (1b) pg_gaussian_loss_kernel: the same scan for a diagonal Gaussian policy (mean per row,
//     state-independent log_std), whose log_std gradient is reduced in a fixed order by
//     pg_gaussian_log_std_grad_kernel (no reference counterpart).
// (1c) gae_kernel + ppo_loss_kernel / ppo_gaussian_loss_kernel: PPO over several epochs of
//     shuffled minibatches (no reference counterpart): GAE(lambda) once per batch, then per
//     minibatch the clipped loss against the rollout policy's log-probs and its gradients,
//     row-parallel, with the batch-side inputs read through an int32 row list.
// (2) sumsq_kernel + adam_kernel: gradient-norm clipping and Adam over ONE flat parameter
//     arena (every trained tensor of a policy is a view into it), no host synchronisation:
//     the clip factor is read from device memory by the Adam kernel.
// The batch forward / backward of the MLP stay on cuBLAS: they are plain [T*E*Np, F] x [F, H]
// library GEMMs with no fusion partner (the loss gradient arrives as a dense tensor), which is
// what cuBLAS is for.
#include <math_constants.h>

#include "wdb_common.cuh"

using namespace wdb;

namespace {

constexpr int kPgThreads = 128;
constexpr float kProbEps = 1.1920928955078125e-07f;   // torch.finfo(float32).eps (clamp_probs)

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) v += __shfl_down_sync(0xffffffffu, v, off);
  return v;
}

// Row blocks through shared memory: the 32 rows a warp works on are ONE contiguous block of
// global memory (rows of 21 / 43 floats: 84 / 172-byte pitches, neither a multiple of the
// sector size), so the warp copies the block with unit-stride accesses into a padded per-warp
// tile (odd pitch: lane r walks row r without bank conflicts) and back.
__device__ __forceinline__ void warp_block_load(float *tile, int pitch, const float *g, int width,
                                                int n_rows, int lane) {
  const int total = n_rows * width;
  const int drow = 32 / width, dcol = 32 - drow * width;
  int row = lane / width, col = lane - row * width;
  int e = lane;
  // four loads in flight per lane before the first shared-memory store waits for one of them
  for (; e + 96 < total; e += 128) {
    const float v0 = g[e], v1 = g[e + 32], v2 = g[e + 64], v3 = g[e + 96];
#define WDB_PUT(V)                                   \
    tile[row * pitch + col] = V;                     \
    row += drow; col += dcol;                        \
    if (col >= width) { col -= width; row++; }
    WDB_PUT(v0) WDB_PUT(v1) WDB_PUT(v2) WDB_PUT(v3)
  }
  for (; e < total; e += 32) {
    const float v = g[e];
    WDB_PUT(v)
  }
#undef WDB_PUT
}
__device__ __forceinline__ void warp_block_store(float *g, const float *tile, int pitch, int width,
                                                 int n_rows, int lane) {
  const int total = n_rows * width;
  const int drow = 32 / width, dcol = 32 - drow * width;
  int row = lane / width, col = lane - row * width;
  for (int e = lane; e < total; e += 32) {
    g[e] = tile[row * pitch + col];
    row += drow; col += dcol;
    if (col >= width) { col -= width; row++; }
  }
}

// sums[0] = sum(-logp * adv), sums[1] = sum((V - R)^2), sums[2] = sum over heads of entropy,
// sums[3] = sum(adv)  (PPO's surrogate at ratio == 1 is -mean(adv))
// Dynamic shared memory: one tile of 32 x (max A | 1) floats per warp.
__global__ void __launch_bounds__(kPgThreads)
pg_loss_kernel(const __grid_constant__ wdb_pg_loss L, int tile_pitch) {
  extern __shared__ float pg_tiles[];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  float *tile = pg_tiles + (size_t)warp * 32 * tile_pitch;
  const long long per_t = (long long)L.n_envs * L.n_agents;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long i0 = i - lane;                          // first index of this warp
  const bool live = i < per_t;
  const int n_rows = (int)max(0ll, min(32ll, per_t - i0));   // rows of this warp that exist
  const int env = live ? (int)(i / L.n_agents) : 0;
  const double inv_m = 1.0 / ((double)L.T * (double)per_t);
  const float inv_mf = (float)inv_m;
  double s_pol = 0.0, s_vf = 0.0, s_ent = 0.0, s_adv = 0.0;
  if (n_rows > 0) {
    float ret = 0.0f;
    for (int t = L.T - 1; t >= 0; t--) {
      const long long idx = (long long)t * per_t + i;
      float adv = 0.0f;
      if (live) {
        const int d = L.done[(long long)t * L.n_envs + env] > 0;
        const float v = L.values[idx];
        // a2c.py:80-93: returns[T-1] = done ? r : V ;  returns[t] = r + (done ? 0 : gamma * next)
        if (t == L.T - 1) ret = d ? L.rewards[idx] : v;
        else ret = L.rewards[idx] + (d ? 0.0f : L.gamma * ret);
        if (L.returns) L.returns[idx] = ret;
        adv = ret - v;
        const float dv = v - ret;
        s_vf += (double)dv * (double)dv;
        s_adv += (double)adv;
        if (L.grad_values) L.grad_values[idx] = 2.0f * L.vf_coeff * dv * inv_mf;
      }
      float logp = 0.0f;
      for (int k = 0; k < L.n_heads; k++) {
        const int A = L.n_actions[k];
        const long long blk = ((long long)t * per_t + i0) * A;   // the warp's 32 x A block
        __syncwarp();
        warp_block_load(tile, tile_pitch, L.probs[k] + blk, A, n_rows, lane);
        __syncwarp();
        if (live) {
          float *p = tile + lane * tile_pitch;                 // this lane's row, overwritten by
          const int a = L.actions[idx * L.n_heads + k];        // its gradient in pass 2
          // torch.distributions.Categorical(probs=p): probs / sum, logits = log(clamp(probs,
          // eps, 1 - eps)); log_prob = logits[a]; entropy = -sum(logits * probs).  torch.clamp's
          // backward passes the gradient for eps <= q <= 1 - eps, both ends inclusive: a
          // near-deterministic float32 row holds q == 1 - eps exactly
          float z = 0.0f;
          for (int j = 0; j < A; j++) z += p[j];
          const float inv_z = 1.0f / z;
          // pass 1: entropy, log-prob and S = sum_i (dL/dq_i) q_i  (q = p / z)
          float ent = 0.0f, S = 0.0f;
          for (int j = 0; j < A; j++) {
            const float q = p[j] * inv_z;
            const bool inside = q >= kProbEps && q <= 1.0f - kProbEps;
            const float lq = logf(fminf(fmaxf(q, kProbEps), 1.0f - kProbEps));
            ent -= lq * q;
            float gq = L.entropy_coeff * (lq + (inside ? 1.0f : 0.0f));   // -c_ent * dH/dq_j
            if (j == a) {
              logp += lq;
              if (inside) gq -= adv / q;                                   // -adv * dlogp/dq_a
            }
            S += gq * q;
          }
          // pass 2: dL/dp_j = (dL/dq_j - S) / z, scaled by 1 / M
          if (L.grad_probs[k]) {
            for (int j = 0; j < A; j++) {
              const float q = p[j] * inv_z;
              const bool inside = q >= kProbEps && q <= 1.0f - kProbEps;
              const float lq = logf(fminf(fmaxf(q, kProbEps), 1.0f - kProbEps));
              float gq = L.entropy_coeff * (lq + (inside ? 1.0f : 0.0f));
              if (j == a && inside) gq -= adv / q;
              p[j] = (gq - S) * inv_mf * inv_z;
            }
          }
          s_ent += (double)ent;
        }
        if (L.grad_probs[k]) {
          __syncwarp();
          warp_block_store(L.grad_probs[k] + blk, tile, tile_pitch, A, n_rows, lane);
        }
      }
      if (live) s_pol += (double)(-logp * adv);
    }
  }
  // block reduction -> 4 double atomics per CTA
  __shared__ double red[4][kPgThreads / 32];
  s_pol = warp_sum(s_pol); s_vf = warp_sum(s_vf); s_ent = warp_sum(s_ent); s_adv = warp_sum(s_adv);
  if (lane == 0) { red[0][warp] = s_pol; red[1][warp] = s_vf; red[2][warp] = s_ent; red[3][warp] = s_adv; }
  __syncthreads();
  if (threadIdx.x < 4) {
    double acc = 0.0;
    for (int w = 0; w < kPgThreads / 32; w++) acc += red[threadIdx.x][w];
    atomicAdd(&L.sums[threadIdx.x], acc);
  }
}

// The Gaussian-policy counterpart of pg_loss_kernel: one thread per (env, agent) row scans T
// backwards; the row's A dimensions stay in registers (fully unrolled over the maximum A).
// sums as pg_loss_kernel; partials[blockIdx.x, k] = sum over the CTA's rows and timesteps of
// adv * (z_k^2 - 1), reduced in a fixed order (shuffle tree, then the warps in order).
constexpr int kGaussMaxA = WDB_PG_GAUSSIAN_MAX_DIM;
constexpr int kGaussThreads = WDB_PG_GAUSSIAN_ROWS_PER_CTA;
constexpr float kHalfLog2Pi = 0.91893853320467274f;   // log(2 pi) / 2

__global__ void __launch_bounds__(kGaussThreads)
pg_gaussian_loss_kernel(const __grid_constant__ wdb_pg_gaussian_loss L) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int A = L.action_dim;
  const long long per_t = (long long)L.n_envs * L.n_agents;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const bool live = i < per_t;
  const int env = live ? (int)(i / L.n_agents) : 0;
  const float inv_mf = (float)(1.0 / ((double)L.T * (double)per_t));
  float ls[kGaussMaxA], inv_std[kGaussMaxA];
  double g_ls[kGaussMaxA];
  float ent = 0.0f;
#pragma unroll
  for (int k = 0; k < kGaussMaxA; k++) {
    ls[k] = k < A ? L.log_std[k] : 0.0f;
    inv_std[k] = expf(-ls[k]);
    g_ls[k] = 0.0;
    if (k < A) ent += ls[k] + (0.5f + kHalfLog2Pi);
  }
  double s_pol = 0.0, s_vf = 0.0, s_ent = 0.0, s_adv = 0.0;
  if (live) {
    float ret = 0.0f;
    for (int t = L.T - 1; t >= 0; t--) {
      const long long idx = (long long)t * per_t + i;
      const int d = L.done[(long long)t * L.n_envs + env] > 0;
      const float v = L.values[idx];
      if (t == L.T - 1) ret = d ? L.rewards[idx] : v;
      else ret = L.rewards[idx] + (d ? 0.0f : L.gamma * ret);
      if (L.returns) L.returns[idx] = ret;
      const float adv = ret - v;
      const float dv = v - ret;
      s_vf += (double)dv * (double)dv;
      s_adv += (double)adv;
      if (L.grad_values) L.grad_values[idx] = 2.0f * L.vf_coeff * dv * inv_mf;
      const float *mu = L.mean + idx * A;
      const float *a = L.actions + idx * A;
      float *gm = L.grad_mean ? L.grad_mean + idx * A : nullptr;
      float logp = 0.0f;
#pragma unroll
      for (int k = 0; k < kGaussMaxA; k++) {
        if (k < A) {
          const float z = (a[k] - mu[k]) * inv_std[k];
          logp += -0.5f * z * z - ls[k] - kHalfLog2Pi;
          // d(-logp * adv) / d mu_k = -adv * z / std;  / d ls_k = -adv * (z^2 - 1)
          if (gm) gm[k] = -adv * z * inv_std[k] * inv_mf;
          g_ls[k] += (double)(adv * (z * z - 1.0f));
        }
      }
      s_pol += (double)(-logp * adv);
      s_ent += (double)ent;
    }
  }
  __shared__ double red[4 + kGaussMaxA][kGaussThreads / 32];
  s_pol = warp_sum(s_pol); s_vf = warp_sum(s_vf); s_ent = warp_sum(s_ent); s_adv = warp_sum(s_adv);
  if (lane == 0) { red[0][warp] = s_pol; red[1][warp] = s_vf; red[2][warp] = s_ent; red[3][warp] = s_adv; }
#pragma unroll
  for (int k = 0; k < kGaussMaxA; k++) {
    if (k < A) {
      const double s = warp_sum(g_ls[k]);
      if (lane == 0) red[4 + k][warp] = s;
    }
  }
  __syncthreads();
  if (threadIdx.x < 4 + A) {
    double acc = 0.0;
    for (int w = 0; w < kGaussThreads / 32; w++) acc += red[threadIdx.x][w];
    if (threadIdx.x < 4) atomicAdd(&L.sums[threadIdx.x], acc);
    else if (L.partials) L.partials[(long long)blockIdx.x * A + threadIdx.x - 4] = acc;
  }
}

// grad_log_std[k] = -(1 / M) * sum over the CTAs, in CTA order, of partials[c, k] - c_ent
// (the entropy term: d mean(H) / d ls_k = 1)
__global__ void pg_gaussian_log_std_grad_kernel(const double *__restrict__ partials, int n_ctas,
                                                int A, double inv_m, float entropy_coeff,
                                                float *__restrict__ grad_log_std) {
  const int k = threadIdx.x;
  if (k >= A) return;
  double acc = 0.0;
  for (int c = 0; c < n_ctas; c++) acc += partials[(long long)c * A + k];
  grad_log_std[k] = (float)(-acc * inv_m - (double)entropy_coeff);
}

// ---- multi-epoch PPO over minibatches: GAE once per batch, then a row-parallel loss ---------
// GAE(lambda) with this repo's bootstrapping convention: one thread per (env, agent) walks T
// backwards; consecutive threads read consecutive rows of a timestep (coalesced).
__global__ void __launch_bounds__(kPgThreads) gae_kernel(const __grid_constant__ wdb_gae_args G) {
  const long long per_t = (long long)G.n_envs * G.n_agents;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= per_t) return;
  const int env = (int)(i / G.n_agents);
  const float gl = G.gamma * G.gae_lambda;
  float adv = 0.0f, v_next = 0.0f;
  for (int t = G.T - 1; t >= 0; t--) {
    const long long idx = (long long)t * per_t + i;
    const int d = G.done[(long long)t * G.n_envs + env] > 0;
    const float r = G.rewards[idx], v = G.values[idx];
    if (t == G.T - 1) {
      adv = d ? r - v : 0.0f;
    } else {
      const float delta = r + (d ? 0.0f : G.gamma * v_next) - v;
      adv = delta + (d ? 0.0f : gl * adv);
    }
    G.advantages[idx] = adv;
    G.value_targets[idx] = adv + v;
    v_next = v;
  }
}

// d loss / d logp of one row, times -B: the weight that replaces `adv` in the A2C gradient.
// PPO: d/d rho of min(rho * A, clamp(rho, 1 - eps, 1 + eps) * A) (torch.minimum splits a tie
// half and half; clamp passes the gradient on its closed interval), times d rho / d logp = rho.
__device__ __forceinline__ float ppo_weight(int ppo, float adv, float rho, float eps) {
  if (!ppo) return adv;
  const float lo = 1.0f - eps, hi = 1.0f + eps;
  const float inside = (rho >= lo && rho <= hi) ? 1.0f : 0.0f;
  const float x = rho * adv, y = fminf(fmaxf(rho, lo), hi) * adv;
  const float g = x < y ? adv : (x > y ? adv * inside : 0.5f * adv + 0.5f * (adv * inside));
  return g * rho;
}

// sums[0..4] of one row into the thread's float64 accumulators (shared by both PPO kernels)
__device__ __forceinline__ void ppo_row_sums(double *s, int ppo, float logp, float old, float rho,
                                             float adv, float eps, float dv, float ent) {
  if (ppo) {
    const float lo = 1.0f - eps, hi = 1.0f + eps;
    s[0] -= (double)fminf(rho * adv, fminf(fmaxf(rho, lo), hi) * adv);
  } else {
    s[0] -= (double)(logp * adv);
  }
  s[1] += (double)dv * (double)dv;
  s[2] += (double)ent;
  s[3] += (double)(old - logp);
  s[4] += fabsf(rho - 1.0f) > eps ? 1.0 : 0.0;
}

// block reduction of the five sums -> 5 double atomics per CTA
template <int kThreads>
__device__ __forceinline__ void ppo_reduce_sums(double *s, double *out) {
  __shared__ double red[5][kThreads / 32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int k = 0; k < 5; k++) {
    const double v = warp_sum(s[k]);
    if (lane == 0) red[k][warp] = v;
  }
  __syncthreads();
  if (threadIdx.x < 5) {
    double acc = 0.0;
    for (int w = 0; w < kThreads / 32; w++) acc += red[threadIdx.x][w];
    atomicAdd(&out[threadIdx.x], acc);
  }
}

// The Categorical minibatch loss: thread b owns minibatch row b; the warp's 32 probability rows
// are one contiguous block (minibatch order) staged through shared memory like pg_loss_kernel.
// Pass 1 over the heads: log-prob and entropy.  Pass 2 (when gradients are asked for): the
// gradient of every head with the row's weight w = -B * d loss / d logp.
__global__ void __launch_bounds__(kPgThreads)
ppo_loss_kernel(const __grid_constant__ wdb_ppo_loss L, int tile_pitch) {
  extern __shared__ float pg_tiles[];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  float *tile = pg_tiles + (size_t)warp * 32 * tile_pitch;
  const long long b = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long b0 = b - lane;
  const bool live = b < L.B;
  const int n_rows = (int)max(0ll, min(32ll, (long long)L.B - b0));
  const bool loss = L.old_log_prob != nullptr;
  const float inv_bf = (float)(1.0 / (double)L.B);
  double s[5] = {0.0, 0.0, 0.0, 0.0, 0.0};
  if (n_rows > 0) {
    const long long row = live ? (L.rows ? (long long)L.rows[b] : b) : 0;
    float logp = 0.0f, ent = 0.0f;
    for (int k = 0; k < L.n_heads; k++) {
      const int A = L.n_actions[k];
      __syncwarp();
      warp_block_load(tile, tile_pitch, L.probs[k] + b0 * A, A, n_rows, lane);
      __syncwarp();
      if (live) {
        // torch.distributions.Categorical(probs=p), as pg_loss_kernel
        const float *p = tile + lane * tile_pitch;
        const int a = L.actions[row * L.n_heads + k];
        float z = 0.0f;
        for (int j = 0; j < A; j++) z += p[j];
        const float inv_z = 1.0f / z;
        for (int j = 0; j < A; j++) {
          const float lq = logf(fminf(fmaxf(p[j] * inv_z, kProbEps), 1.0f - kProbEps));
          ent -= lq * (p[j] * inv_z);
          if (j == a) logp += lq;
        }
      }
    }
    if (live && L.log_prob) L.log_prob[b] = logp;
    float w = 0.0f;
    if (loss && live) {
      const float old = L.old_log_prob[row], adv = L.advantages[row];
      const float rho = expf(logp - old);
      const float dv = L.values[b] - L.value_targets[row];
      w = ppo_weight(L.ppo, adv, rho, L.clip_param);
      ppo_row_sums(s, L.ppo, logp, old, rho, adv, L.clip_param, dv, ent);
      if (L.grad_values) L.grad_values[b] = 2.0f * L.vf_coeff * dv * inv_bf;
    }
    for (int k = 0; k < L.n_heads; k++) {
      if (!L.grad_probs[k]) continue;
      const int A = L.n_actions[k];
      if (L.n_heads > 1) {               // one head: the tile still holds its rows
        __syncwarp();
        warp_block_load(tile, tile_pitch, L.probs[k] + b0 * A, A, n_rows, lane);
        __syncwarp();
      }
      if (live) {
        float *p = tile + lane * tile_pitch;
        const int a = L.actions[row * L.n_heads + k];
        float z = 0.0f;
        for (int j = 0; j < A; j++) z += p[j];
        const float inv_z = 1.0f / z;
        float S = 0.0f;
        for (int j = 0; j < A; j++) {
          const float q = p[j] * inv_z;
          const bool inside = q >= kProbEps && q <= 1.0f - kProbEps;
          const float lq = logf(fminf(fmaxf(q, kProbEps), 1.0f - kProbEps));
          float gq = L.entropy_coeff * (lq + (inside ? 1.0f : 0.0f));
          if (j == a && inside) gq -= w / q;
          S += gq * q;
        }
        for (int j = 0; j < A; j++) {
          const float q = p[j] * inv_z;
          const bool inside = q >= kProbEps && q <= 1.0f - kProbEps;
          const float lq = logf(fminf(fmaxf(q, kProbEps), 1.0f - kProbEps));
          float gq = L.entropy_coeff * (lq + (inside ? 1.0f : 0.0f));
          if (j == a && inside) gq -= w / q;
          p[j] = (gq - S) * inv_bf * inv_z;
        }
      }
      __syncwarp();
      warp_block_store(L.grad_probs[k] + b0 * A, tile, tile_pitch, A, n_rows, lane);
    }
  }
  if (loss) ppo_reduce_sums<kPgThreads>(s, L.sums);
}

// The diagonal-Gaussian minibatch loss: thread b owns minibatch row b, its A dimensions in
// registers.  partials[blockIdx.x, k] = sum over the CTA's rows of w * (z_k^2 - 1), reduced in
// a fixed order; pg_gaussian_log_std_grad_kernel turns them into the log_std gradient.
__global__ void __launch_bounds__(kGaussThreads)
ppo_gaussian_loss_kernel(const __grid_constant__ wdb_ppo_gaussian_loss L) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int A = L.action_dim;
  const long long b = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const bool live = b < L.B;
  const bool loss = L.old_log_prob != nullptr;
  const float inv_bf = (float)(1.0 / (double)L.B);
  float ls[kGaussMaxA], inv_std[kGaussMaxA];
  double g_ls[kGaussMaxA];
  float ent = 0.0f;
#pragma unroll
  for (int k = 0; k < kGaussMaxA; k++) {
    ls[k] = k < A ? L.log_std[k] : 0.0f;
    inv_std[k] = expf(-ls[k]);
    g_ls[k] = 0.0;
    if (k < A) ent += ls[k] + (0.5f + kHalfLog2Pi);
  }
  double s[5] = {0.0, 0.0, 0.0, 0.0, 0.0};
  if (live) {
    const long long row = L.rows ? (long long)L.rows[b] : b;
    const float *mu = L.mean + b * A;
    const float *a = L.actions + row * A;
    float z[kGaussMaxA];
    float logp = 0.0f;
#pragma unroll
    for (int k = 0; k < kGaussMaxA; k++) {
      if (k < A) {
        z[k] = (a[k] - mu[k]) * inv_std[k];
        logp += -0.5f * z[k] * z[k] - ls[k] - kHalfLog2Pi;
      }
    }
    if (L.log_prob) L.log_prob[b] = logp;
    if (loss) {
      const float old = L.old_log_prob[row], adv = L.advantages[row];
      const float rho = expf(logp - old);
      const float dv = L.values[b] - L.value_targets[row];
      const float w = ppo_weight(L.ppo, adv, rho, L.clip_param);
      ppo_row_sums(s, L.ppo, logp, old, rho, adv, L.clip_param, dv, ent);
      if (L.grad_values) L.grad_values[b] = 2.0f * L.vf_coeff * dv * inv_bf;
      float *gm = L.grad_mean ? L.grad_mean + b * A : nullptr;
#pragma unroll
      for (int k = 0; k < kGaussMaxA; k++) {
        if (k < A) {
          // d(-logp * w) / d mu_k = -w * z / std;  / d ls_k = -w * (z^2 - 1)
          if (gm) gm[k] = -w * z[k] * inv_std[k] * inv_bf;
          g_ls[k] += (double)(w * (z[k] * z[k] - 1.0f));
        }
      }
    }
  }
  if (!loss) return;
  ppo_reduce_sums<kGaussThreads>(s, L.sums);
  __shared__ double red[kGaussMaxA][kGaussThreads / 32];
#pragma unroll
  for (int k = 0; k < kGaussMaxA; k++) {
    if (k < A) {
      const double v = warp_sum(g_ls[k]);
      if (lane == 0) red[k][warp] = v;
    }
  }
  __syncthreads();
  if (threadIdx.x < A && L.partials) {
    double acc = 0.0;
    for (int w = 0; w < kGaussThreads / 32; w++) acc += red[threadIdx.x][w];
    L.partials[(long long)blockIdx.x * A + threadIdx.x] = acc;
  }
}

// sum of squares of a flat float buffer -> *out (double, zeroed by the caller)
__global__ void __launch_bounds__(256) sumsq_kernel(const float *__restrict__ g, long long n,
                                                    double *out) {
  double acc = 0.0;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n;
       i += (long long)gridDim.x * blockDim.x) {
    const float v = g[i];
    acc += (double)v * (double)v;
  }
  acc = warp_sum(acc);
  __shared__ double red[8];
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double s = 0.0;
    for (int w = 0; w < 8; w++) s += red[w];
    atomicAdd(out, s);
  }
}

// torch.optim.Adam (no weight decay, no amsgrad) on a flat arena; the gradient is first scaled
// by clip = min(1, max_norm / (norm + 1e-6)) like torch.nn.utils.clip_grad_norm_ (the scaled
// gradient is written back: callers that log the clipped gradient see the same values)
__global__ void __launch_bounds__(256)
adam_kernel(float *__restrict__ p, float *__restrict__ g, float *__restrict__ m,
            float *__restrict__ v, long long n, float lr, float beta1, float beta2, float eps,
            float bias1, float bias2_sqrt, float max_norm, const double *sumsq) {
  float clip = 1.0f;
  if (max_norm > 0.0f && sumsq) {
    const float norm = (float)sqrt(*sumsq);
    clip = fminf(1.0f, max_norm / (norm + 1.0e-6f));
  }
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float gi = g[i] * clip;
  g[i] = gi;
  const float mi = beta1 * m[i] + (1.0f - beta1) * gi;      // lerp form of torch's foreach Adam
  const float vi = beta2 * v[i] + (1.0f - beta2) * gi * gi;
  m[i] = mi;
  v[i] = vi;
  const float denom = sqrtf(vi) / bias2_sqrt + eps;
  p[i] = p[i] - (lr / bias1) * (mi / denom);
}


// ---- elementwise pieces of the MLP's training forward / backward (the GEMMs stay on cuBLAS;
// these replace the separate torch kernels -- and tensor passes -- between them) ------------
// logits [M, pitch] (two action heads and the value column of ONE GEMM) -> softmax per head
// into dense probs0 / probs1, value column into values.  A warp stages its 32 rows through a
// padded shared-memory tile (warp_block_load / _store): unit-stride global accesses.
constexpr int kRowThreads = 128;
// the per-head softmax of one staged row (heads_softmax_masked_kernel; heads_softmax_kernel
// keeps its own copy of these lines so that its machine code stays as it was)
__device__ __forceinline__ void softmax_heads_row(float *row, int A0, int A1) {
  for (int h = 0; h < 2; h++) {
    const int n = h ? A1 : A0;
    float *x = row + (h ? A0 : 0);
    if (n == 0) continue;
    float mx = x[0];
    for (int j = 1; j < n; j++) mx = fmaxf(mx, x[j]);
    float sum = 0.0f;
    for (int j = 0; j < n; j++) { const float e = expf(x[j] - mx); x[j] = e; sum += e; }
    const float inv = 1.0f / sum;
    for (int j = 0; j < n; j++) x[j] *= inv;
  }
}

__global__ void __launch_bounds__(kRowThreads)
heads_softmax_kernel(const float *__restrict__ z, long long M, int A0, int A1, int ld,
                     float *__restrict__ p0, float *__restrict__ p1, float *__restrict__ values,
                     int tile_pitch) {
  extern __shared__ float row_tiles[];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  float *tile = row_tiles + (size_t)warp * 32 * tile_pitch;
  const long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long r0 = r - lane;
  const int n_rows = (int)max(0ll, min(32ll, M - r0));
  if (n_rows == 0) return;
  const bool live = r < M;
  warp_block_load(tile, tile_pitch, z + r0 * ld, ld, n_rows, lane);
  __syncwarp();
  float *row = tile + lane * tile_pitch;
  if (live) {
    for (int h = 0; h < 2; h++) {
      const int n = h ? A1 : A0;
      float *x = row + (h ? A0 : 0);
      if (n == 0) continue;
      float mx = x[0];
      for (int j = 1; j < n; j++) mx = fmaxf(mx, x[j]);
      float sum = 0.0f;
      for (int j = 0; j < n; j++) { const float e = expf(x[j] - mx); x[j] = e; sum += e; }
      const float inv = 1.0f / sum;
      for (int j = 0; j < n; j++) x[j] *= inv;
    }
    values[r] = row[A0 + A1];
  }
  __syncwarp();
  warp_block_store(p0 + r0 * A0, tile, tile_pitch, A0, n_rows, lane);
  if (A1 > 0) warp_block_store(p1 + r0 * A1, tile + A0, tile_pitch, A1, n_rows, lane);
}

// the same with an action mask [M, mask_ld]: logit + (1 - m) * -1e20 (FullyConnected's
// apply_logit_mask, fp32) before each head's max; the warp's mask rows are staged in a
// second tile like the logits
__global__ void __launch_bounds__(kRowThreads)
heads_softmax_masked_kernel(const float *__restrict__ z, long long M, int A0, int A1, int ld,
                            const float *__restrict__ mask, int mask_ld,
                            float *__restrict__ p0, float *__restrict__ p1,
                            float *__restrict__ values, int tile_pitch) {
  extern __shared__ float row_tiles[];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  float *tile = row_tiles + (size_t)warp * 64 * tile_pitch;
  float *tm = tile + 32 * tile_pitch;
  const long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long r0 = r - lane;
  const int n_rows = (int)max(0ll, min(32ll, M - r0));
  if (n_rows == 0) return;
  const bool live = r < M;
  warp_block_load(tile, tile_pitch, z + r0 * ld, ld, n_rows, lane);
  warp_block_load(tm, tile_pitch, mask + r0 * mask_ld, mask_ld, n_rows, lane);
  __syncwarp();
  float *row = tile + lane * tile_pitch;
  if (live) {
    const float *m = tm + lane * tile_pitch;
    for (int j = 0; j < A0 + A1; j++) row[j] = __fadd_rn(row[j], __fmul_rn(1.0f - m[j], -1.0e20f));
    softmax_heads_row(row, A0, A1);
    values[r] = row[A0 + A1];
  }
  __syncwarp();
  warp_block_store(p0 + r0 * A0, tile, tile_pitch, A0, n_rows, lane);
  if (A1 > 0) warp_block_store(p1 + r0 * A1, tile + A0, tile_pitch, A1, n_rows, lane);
}

// d(logits) from d(probs): dz_j = p_j (g_j - sum_k g_k p_k) per head; value column = gv;
// the padding columns of the pitch = 0
__global__ void __launch_bounds__(kRowThreads)
heads_softmax_backward_kernel(const float *__restrict__ p0, const float *__restrict__ p1,
                              const float *__restrict__ g0, const float *__restrict__ g1,
                              const float *__restrict__ gv, long long M, int A0, int A1,
                              int ld, float *__restrict__ dz, int tile_pitch) {
  extern __shared__ float row_tiles[];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  // two tiles per warp: probabilities (becomes dz, full pitch) and incoming gradients
  float *tp = row_tiles + (size_t)warp * 64 * tile_pitch;
  float *tg = tp + 32 * tile_pitch;
  const long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long r0 = r - lane;
  const int n_rows = (int)max(0ll, min(32ll, M - r0));
  if (n_rows == 0) return;
  const bool live = r < M;
  warp_block_load(tp, tile_pitch, p0 + r0 * A0, A0, n_rows, lane);
  if (A1 > 0) warp_block_load(tp + A0, tile_pitch, p1 + r0 * A1, A1, n_rows, lane);
  if (g0) warp_block_load(tg, tile_pitch, g0 + r0 * A0, A0, n_rows, lane);
  if (g1 && A1 > 0) warp_block_load(tg + A0, tile_pitch, g1 + r0 * A1, A1, n_rows, lane);
  __syncwarp();
  if (live) {
    float *prow = tp + lane * tile_pitch;
    const float *grow = tg + lane * tile_pitch;
    for (int h = 0; h < 2; h++) {
      const int n = h ? A1 : A0;
      if (n == 0) continue;
      float *p = prow + (h ? A0 : 0);
      const float *g = grow + (h ? A0 : 0);
      if (!(h ? g1 : g0)) {                       // this head received no gradient
        for (int j = 0; j < n; j++) p[j] = 0.0f;
        continue;
      }
      float dot = 0.0f;
      for (int j = 0; j < n; j++) dot += g[j] * p[j];
      for (int j = 0; j < n; j++) p[j] = p[j] * (g[j] - dot);
    }
    prow[A0 + A1] = gv ? gv[r] : 0.0f;
    for (int j = A0 + A1 + 1; j < ld; j++) prow[j] = 0.0f;
  }
  __syncwarp();
  warp_block_store(dz + r0 * ld, tp, tile_pitch, ld, n_rows, lane);
}

// ReLU backward in place + the bias gradient of the layer: dh[r, c] = h[r, c] > 0 ? dh[r, c] : 0,
// partial[blockIdx.x, c] = sum over this CTA's rows (the caller adds the partials: no atomics,
// deterministic).  float4 columns: a 256-thread CTA covers 1024 / H whole rows per iteration,
// four iterations unrolled with all loads ahead of the stores (the kernel is a pure stream:
// 12 bytes per element, what matters is bytes in flight).
__global__ void __launch_bounds__(256)
relu_backward_bias_kernel(float *__restrict__ dh, const float *__restrict__ h, long long M, int H,
                          int rows_per_cta, float *__restrict__ partial) {
  const int cpr = H >> 2;                          // float4 columns per row
  const int rpi = blockDim.x / cpr;                // rows per iteration
  const int sub = threadIdx.x / cpr, c4 = threadIdx.x - sub * cpr;
  const long long r0 = (long long)blockIdx.x * rows_per_cta;
  const long long r1 = min(M, r0 + rows_per_cta);
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
  if (sub < rpi) {
    float4 *d4 = reinterpret_cast<float4 *>(dh);
    const float4 *h4 = reinterpret_cast<const float4 *>(h);
    long long r = r0 + sub;
    for (; r + 3ll * rpi < r1; r += 4ll * rpi) {
      float4 a[4], g[4];
#pragma unroll
      for (int u = 0; u < 4; u++) {
        const long long i = (r + (long long)u * rpi) * cpr + c4;
        a[u] = h4[i];
        g[u] = d4[i];
      }
#pragma unroll
      for (int u = 0; u < 4; u++) {
        const long long i = (r + (long long)u * rpi) * cpr + c4;
        g[u].x = a[u].x > 0.0f ? g[u].x : 0.0f; g[u].y = a[u].y > 0.0f ? g[u].y : 0.0f;
        g[u].z = a[u].z > 0.0f ? g[u].z : 0.0f; g[u].w = a[u].w > 0.0f ? g[u].w : 0.0f;
        d4[i] = g[u];
        acc.x += g[u].x; acc.y += g[u].y; acc.z += g[u].z; acc.w += g[u].w;
      }
    }
    for (; r < r1; r += rpi) {
      const long long i = r * cpr + c4;
      const float4 a = h4[i];
      float4 g = d4[i];
      g.x = a.x > 0.0f ? g.x : 0.0f; g.y = a.y > 0.0f ? g.y : 0.0f;
      g.z = a.z > 0.0f ? g.z : 0.0f; g.w = a.w > 0.0f ? g.w : 0.0f;
      d4[i] = g;
      acc.x += g.x; acc.y += g.y; acc.z += g.z; acc.w += g.w;
    }
  }
  // column sums over the CTA's sub-rows (fixed order: deterministic)
  __shared__ float4 red[256];
  red[threadIdx.x] = acc;
  __syncthreads();
  if (sub == 0 && c4 < cpr) {
    float4 s = red[c4];
    for (int k = 1; k < rpi; k++) {
      const float4 v = red[k * cpr + c4];
      s.x += v.x; s.y += v.y; s.z += v.z; s.w += v.w;
    }
    reinterpret_cast<float4 *>(partial)[(long long)blockIdx.x * cpr + c4] = s;
  }
}

// same, scalar columns (widths that are not a multiple of 4 / unaligned bases)
__global__ void __launch_bounds__(256)
relu_backward_bias_scalar_kernel(float *__restrict__ dh, const float *__restrict__ h, long long M,
                                 int H, int rows_per_cta, float *__restrict__ partial) {
  const long long r0 = (long long)blockIdx.x * rows_per_cta;
  const long long r1 = min(M, r0 + rows_per_cta);
  for (int c = threadIdx.x; c < H; c += blockDim.x) {
    float acc = 0.0f;
    for (long long r = r0; r < r1; r++) {
      const long long i = r * H + c;
      const float v = h[i] > 0.0f ? dh[i] : 0.0f;
      dh[i] = v;
      acc += v;
    }
    partial[(long long)blockIdx.x * H + c] = acc;
  }
}


// rows of `width` floats -> rows of `pitch` >= width floats, zero-filled (the 16-byte-aligned
// copy of the observations the first-layer GEMMs read); one thread per output element
__global__ void __launch_bounds__(256)
pad_rows_kernel(const float *__restrict__ src, long long rows, int width, int pitch,
                float *__restrict__ dst) {
  const long long n = rows * pitch;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n;
       i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / pitch;
    const int c = (int)(i - r * pitch);
    dst[i] = c < width ? src[r * width + c] : 0.0f;
  }
}

}  // namespace

namespace {

constexpr size_t kRowSmemLimit = 200 * 1024;   // dynamic shared memory the row-tile kernels opt into

// shared memory of pg_loss_kernel: one 32-row tile per warp of the widest head (odd pitch);
// 0 for a head set the kernel does not take
size_t pg_loss_smem(int n_heads, const int *n_actions, int *tile_pitch) {
  if (n_heads < 1 || n_heads > 4 || !n_actions) return 0;
  int amax = 1;
  for (int k = 0; k < n_heads; k++) {
    if (n_actions[k] < 1) return 0;
    amax = n_actions[k] > amax ? n_actions[k] : amax;
  }
  const int pitch = amax | 1;                                   // odd: no bank conflicts
  const size_t smem = (size_t)(kPgThreads / 32) * 32 * pitch * sizeof(float);
  if (smem > kRowSmemLimit) return 0;
  if (tile_pitch) *tile_pitch = pitch;
  return smem;
}

// shared memory of the heads softmax forward (tiles == 1) / backward (tiles == 2) at a logits
// pitch; 0 for a shape the kernel does not take
size_t heads_softmax_smem(int A0, int A1, int pitch, int tiles) {
  if (A0 < 1 || A1 < 0 || pitch < A0 + A1 + 1) return 0;
  const size_t smem = (size_t)(kRowThreads / 32) * 32 * tiles * (pitch | 1) * sizeof(float);
  return smem > kRowSmemLimit ? 0 : smem;
}

}  // namespace

WDB_API int wdb_pg_loss_supported(int n_heads, const int *n_actions) {
  return pg_loss_smem(n_heads, n_actions, nullptr) > 0;
}

WDB_API int wdb_pg_gaussian_loss_supported(int action_dim) {
  return action_dim >= 1 && action_dim <= kGaussMaxA;
}

WDB_API int wdb_pg_gaussian_loss_and_grads(void *stream, const wdb_pg_gaussian_loss *l) {
  if (!l || l->T < 1 || l->n_envs < 1 || l->n_agents < 1 ||
      !wdb_pg_gaussian_loss_supported(l->action_dim))
    return (int)cudaErrorInvalidValue;
  if (!l->mean || !l->log_std || !l->values || !l->actions || !l->rewards || !l->done ||
      !l->sums || (l->grad_log_std && !l->partials))
    return (int)cudaErrorInvalidValue;
  const long long n = (long long)l->n_envs * l->n_agents;
  const int grid = (int)((n + kGaussThreads - 1) / kGaussThreads);
  pg_gaussian_loss_kernel<<<grid, kGaussThreads, 0, as_stream(stream)>>>(*l);
  int err = finish_launch();
  if (err || !l->grad_log_std) return err;
  pg_gaussian_log_std_grad_kernel<<<1, 32, 0, as_stream(stream)>>>(
      l->partials, grid, l->action_dim, 1.0 / ((double)l->T * (double)n), l->entropy_coeff,
      l->grad_log_std);
  return finish_launch();
}

WDB_API int wdb_gae(void *stream, const wdb_gae_args *g) {
  if (!g || g->T < 1 || g->n_envs < 1 || g->n_agents < 1 || !g->rewards || !g->values ||
      !g->done || !g->advantages || !g->value_targets)
    return (int)cudaErrorInvalidValue;
  const long long n = (long long)g->n_envs * g->n_agents;
  gae_kernel<<<(unsigned)((n + kPgThreads - 1) / kPgThreads), kPgThreads, 0,
               as_stream(stream)>>>(*g);
  return finish_launch();
}

WDB_API int wdb_ppo_loss_supported(int n_heads, const int *n_actions) {
  return pg_loss_smem(n_heads, n_actions, nullptr) > 0;
}

WDB_API int wdb_ppo_gaussian_loss_supported(int action_dim) {
  return action_dim >= 1 && action_dim <= kGaussMaxA;
}

// The loss mode (old_log_prob given) needs every per-row input and the sums; the log-prob
// pre-pass (old_log_prob NULL) needs log_prob and takes no gradient outputs.
static bool ppo_common_ok(int B, const void *old_log_prob, const float *log_prob,
                          const float *values, const float *advantages,
                          const float *value_targets, const double *sums, bool any_grad) {
  if (B < 1) return false;
  if (!old_log_prob) return log_prob && !any_grad;
  return values && advantages && value_targets && sums;
}

WDB_API int wdb_ppo_loss_and_grads(void *stream, const wdb_ppo_loss *l) {
  if (!l) return (int)cudaErrorInvalidValue;
  int pitch = 0;
  const size_t smem = pg_loss_smem(l->n_heads, l->n_actions, &pitch);
  if (!smem || !l->actions) return (int)cudaErrorInvalidValue;
  bool any_grad = l->grad_values != nullptr;
  for (int k = 0; k < l->n_heads; k++) {
    if (!l->probs[k]) return (int)cudaErrorInvalidValue;
    any_grad = any_grad || l->grad_probs[k];
  }
  if (!ppo_common_ok(l->B, l->old_log_prob, l->log_prob, l->values, l->advantages,
                     l->value_targets, l->sums, any_grad))
    return (int)cudaErrorInvalidValue;
  static size_t configured = 48 * 1024;
  if (smem > configured) {
    cudaError_t e = cudaFuncSetAttribute(ppo_loss_kernel,
                                         cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return (int)e;
    configured = smem;
  }
  ppo_loss_kernel<<<(unsigned)(((long long)l->B + kPgThreads - 1) / kPgThreads), kPgThreads, smem,
                    as_stream(stream)>>>(*l, pitch);
  return finish_launch();
}

WDB_API int wdb_ppo_gaussian_loss_and_grads(void *stream, const wdb_ppo_gaussian_loss *l) {
  if (!l || !wdb_ppo_gaussian_loss_supported(l->action_dim) || !l->mean || !l->log_std ||
      !l->actions)
    return (int)cudaErrorInvalidValue;
  const bool any_grad = l->grad_mean || l->grad_log_std || l->grad_values;
  if (!ppo_common_ok(l->B, l->old_log_prob, l->log_prob, l->values, l->advantages,
                     l->value_targets, l->sums, any_grad) ||
      (l->grad_log_std && !l->partials))
    return (int)cudaErrorInvalidValue;
  const int grid = (int)(((long long)l->B + kGaussThreads - 1) / kGaussThreads);
  ppo_gaussian_loss_kernel<<<grid, kGaussThreads, 0, as_stream(stream)>>>(*l);
  int err = finish_launch();
  if (err || !l->grad_log_std) return err;
  pg_gaussian_log_std_grad_kernel<<<1, 32, 0, as_stream(stream)>>>(
      l->partials, grid, l->action_dim, 1.0 / (double)l->B, l->entropy_coeff, l->grad_log_std);
  return finish_launch();
}

WDB_API int wdb_heads_softmax_supported(int A0, int A1, int pitch) {
  return heads_softmax_smem(A0, A1, pitch, 1) > 0 && heads_softmax_smem(A0, A1, pitch, 2) > 0;
}

WDB_API int wdb_pg_loss_and_grads(void *stream, const wdb_pg_loss *l) {
  if (!l || l->T < 1 || l->n_envs < 1 || l->n_agents < 1) return (int)cudaErrorInvalidValue;
  int pitch = 0;
  const size_t smem = pg_loss_smem(l->n_heads, l->n_actions, &pitch);
  if (!smem) return (int)cudaErrorInvalidValue;
  if (!l->values || !l->actions || !l->rewards || !l->done || !l->sums)
    return (int)cudaErrorInvalidValue;
  for (int k = 0; k < l->n_heads; k++)
    if (!l->probs[k]) return (int)cudaErrorInvalidValue;
  const long long n = (long long)l->n_envs * l->n_agents;
  const int grid = (int)((n + kPgThreads - 1) / kPgThreads);
  static size_t configured = 48 * 1024;
  if (smem > configured) {
    cudaError_t e = cudaFuncSetAttribute(pg_loss_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         (int)smem);
    if (e != cudaSuccess) return (int)e;
    configured = smem;
  }
  pg_loss_kernel<<<grid, kPgThreads, smem, as_stream(stream)>>>(*l, pitch);
  return finish_launch();
}

WDB_API int wdb_grad_sumsq(void *stream, const float *grads, long long n, double *out) {
  if (!grads || !out || n < 1) return (int)cudaErrorInvalidValue;
  long long blocks = (n + 256 * 8 - 1) / (256 * 8);
  if (blocks > 4 * kNumSMs) blocks = 4 * kNumSMs;
  if (blocks < 1) blocks = 1;
  sumsq_kernel<<<(int)blocks, 256, 0, as_stream(stream)>>>(grads, n, out);
  return finish_launch();
}

WDB_API int wdb_adam_step(void *stream, float *params, float *grads, float *exp_avg,
                          float *exp_avg_sq, long long n, float lr, float beta1, float beta2,
                          float eps, int step, float max_grad_norm, const double *grad_sumsq) {
  if (!params || !grads || !exp_avg || !exp_avg_sq || n < 1 || step < 1)
    return (int)cudaErrorInvalidValue;
  if (max_grad_norm > 0.0f && !grad_sumsq) return (int)cudaErrorInvalidValue;
  const float bias1 = 1.0f - powf(beta1, (float)step);
  const float bias2_sqrt = sqrtf(1.0f - powf(beta2, (float)step));
  adam_kernel<<<(int)((n + 255) / 256), 256, 0, as_stream(stream)>>>(
      params, grads, exp_avg, exp_avg_sq, n, lr, beta1, beta2, eps, bias1, bias2_sqrt,
      max_grad_norm, grad_sumsq);
  return finish_launch();
}

WDB_API int wdb_heads_softmax(void *stream, const float *logits, long long rows, int A0, int A1,
                              int pitch, float *probs0, float *probs1, float *values) {
  const size_t smem = heads_softmax_smem(A0, A1, pitch, 1);
  if (!logits || !probs0 || !values || rows < 1 || !smem || (A1 > 0 && !probs1))
    return (int)cudaErrorInvalidValue;
  const int tp = pitch | 1;
  {
    static size_t configured = 48 * 1024;
    if (smem > configured) {
      cudaError_t e = cudaFuncSetAttribute(heads_softmax_kernel,
                                           cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
      if (e != cudaSuccess) return (int)e;
      configured = smem;
    }
  }
  heads_softmax_kernel<<<(unsigned)((rows + kRowThreads - 1) / kRowThreads), kRowThreads, smem,
                         as_stream(stream)>>>(logits, rows, A0, A1, pitch, probs0, probs1, values,
                                              tp);
  return finish_launch();
}

WDB_API int wdb_heads_softmax_masked(void *stream, const float *logits, long long rows, int A0,
                                     int A1, int pitch, const float *mask, int mask_pitch,
                                     float *probs0, float *probs1, float *values) {
  // two row tiles per warp (logits, mask): the backward's shared memory
  const size_t smem = heads_softmax_smem(A0, A1, pitch, 2);
  if (!logits || !mask || !probs0 || !values || rows < 1 || !smem || (A1 > 0 && !probs1) ||
      mask_pitch < A0 + A1 || mask_pitch > pitch)
    return (int)cudaErrorInvalidValue;
  const int tp = pitch | 1;
  {
    static size_t configured = 48 * 1024;
    if (smem > configured) {
      cudaError_t e = cudaFuncSetAttribute(heads_softmax_masked_kernel,
                                           cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
      if (e != cudaSuccess) return (int)e;
      configured = smem;
    }
  }
  heads_softmax_masked_kernel<<<(unsigned)((rows + kRowThreads - 1) / kRowThreads), kRowThreads,
                                smem, as_stream(stream)>>>(logits, rows, A0, A1, pitch, mask,
                                                           mask_pitch, probs0, probs1, values, tp);
  return finish_launch();
}

WDB_API int wdb_heads_softmax_backward(void *stream, const float *probs0, const float *probs1,
                                       const float *grad_probs0, const float *grad_probs1,
                                       const float *grad_values, long long rows, int A0, int A1,
                                       int pitch, float *grad_logits) {
  const size_t smem = heads_softmax_smem(A0, A1, pitch, 2);
  if (!probs0 || !grad_logits || rows < 1 || !smem || (A1 > 0 && !probs1))
    return (int)cudaErrorInvalidValue;
  const int tp = pitch | 1;
  {
    static size_t configured = 48 * 1024;
    if (smem > configured) {
      cudaError_t e = cudaFuncSetAttribute(heads_softmax_backward_kernel,
                                           cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
      if (e != cudaSuccess) return (int)e;
      configured = smem;
    }
  }
  heads_softmax_backward_kernel<<<(unsigned)((rows + kRowThreads - 1) / kRowThreads), kRowThreads,
                                  smem, as_stream(stream)>>>(
      probs0, probs1, grad_probs0, grad_probs1, grad_values, rows, A0, A1, pitch, grad_logits, tp);
  return finish_launch();
}

WDB_API int wdb_relu_backward_bias_rows(long long rows) {
  // rows handled by one CTA: enough CTAs to fill the GPU several times, few enough partials
  long long per = (rows + 8 * kNumSMs - 1) / (8 * kNumSMs);
  if (per < 64) per = 64;
  return (int)per;
}

WDB_API int wdb_relu_backward_bias(void *stream, float *grad_hidden, const float *hidden,
                                   long long rows, int width, float *partial_bias_grads) {
  if (!grad_hidden || !hidden || !partial_bias_grads || rows < 1 || width < 1)
    return (int)cudaErrorInvalidValue;
  const int per = wdb_relu_backward_bias_rows(rows);
  const long long ctas = (rows + per - 1) / per;
  const bool vec = (width % 4 == 0) && (width / 4 <= 256) &&
                   ((reinterpret_cast<uintptr_t>(grad_hidden) | reinterpret_cast<uintptr_t>(hidden) |
                     reinterpret_cast<uintptr_t>(partial_bias_grads)) & 15) == 0;
  if (vec)
    relu_backward_bias_kernel<<<(unsigned)ctas, 256, 0, as_stream(stream)>>>(
        grad_hidden, hidden, rows, width, per, partial_bias_grads);
  else
    relu_backward_bias_scalar_kernel<<<(unsigned)ctas, 256, 0, as_stream(stream)>>>(
        grad_hidden, hidden, rows, width, per, partial_bias_grads);
  return finish_launch();
}

WDB_API int wdb_pad_rows(void *stream, const float *src, long long rows, int width, int pitch,
                         float *dst) {
  if (!src || !dst || rows < 1 || width < 1 || pitch < width) return (int)cudaErrorInvalidValue;
  long long blocks = (rows * pitch + 255) / 256;
  if (blocks > 32ll * kNumSMs) blocks = 32ll * kNumSMs;
  pad_rows_kernel<<<(unsigned)blocks, 256, 0, as_stream(stream)>>>(src, rows, width, pitch, dst);
  return finish_launch();
}
