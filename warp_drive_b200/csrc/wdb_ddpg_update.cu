// wdb_ddpg_update.cu -- every gradient of one DDPG update of one policy in one launch, read in
// place from the replay ring, plus a fixed-order reduction of the per-CTA partials into the
// gradient arena (include/wdb200.h, wdb_ddpg_update).
//
// Replaces TrainerDDPG._update_model_params' torch autograd body (trainer_ddpg.py:380-420 of
// the reference): five MLP forwards over the whole unrolled ring, the n-step returns
// (ddpg.py:62-79), both losses and two backward passes -- over a hundred small launches.
//
// Per tile of kRows loss rows (row g = logical slot i * E * Np + agent row n), in shared
// memory and in this order:
//   target actor, target critic on obs at slot i + n_step (the last window: capacity - 1)
//   -> the bootstrap value; critic on (obs, actions) -> Q; actor on obs -> pi; critic on
//   (obs, pi) -> J; n-step return R; dL/dQ = 2 (Q - R) / M, dL/dJ = -1 / M; back through the
//   critic on both paths (the reference's actor_loss.backward() also reaches the critic), the
//   J path on to the action inputs, the tanh head and the actor.
// The weight gradients of a tile are added to per-CTA accumulators in shared memory; each CTA
// writes them once as its partial, and the second kernel sums the partials in CTA order.  No
// float atomics: an update is bit-reproducible.
//
// Why no tensor cores: the reasons of wdb_sa_rollout.cu -- the networks are tiny (3 or 4 ->
// 64 -> 64 -> 1), all four fit shared memory, and the torch reference is float32 (TF32 off).
//
// Thread layout (256 threads, 16-row tiles): forward and input-gradient steps give each
// thread one output column and four rows (one float4 weight load feeds sixteen FMAs);
// weight-gradient steps give each thread one input column and sixteen output rows.
//
// TD3 (wdb_td3_critic_update / wdb_td3_actor_update) runs on the same tile primitives, Plan
// layout and reduction, as two passes of two launches each:
//   critic pass, per tile: target actor on obs' -> a' = clamp(pi' + clamp(sigma scale eps,
//     -c scale, c scale), bias - scale, bias + scale); both target critics on (obs', a') ->
//     min -> the n-step return R; Q1 and Q2 on (obs, actions); dL/dQk = 2 (Qk - R) / M; back
//     through each critic into its own gradient block (no actor-loss term).
//   actor pass, per tile: actor on obs -> pi; Q1 on (obs, pi) -> J; dL/dJ = -1 / M back
//     through Q1 to its action inputs only (no critic weight gradient), the tanh head and the
//     actor.
//
// Replay buffer (wdb_*_update_sampled): each of the five passes also runs over B sampled
// windows of a long ring, row g = windows[g] instead of (g / EN, g % EN) -- the same kernel
// template instantiated for the other row source ("loss rows" below).
#include <type_traits>

#include "wdb_common.cuh"
#include "wdb_update_tiles.cuh"          // Plan, the layer steps, SampledRows, the reduction
#include "wdb_dqn_pass.cuh"              // DQN's tile body and plan
#include "wdb_sac_terms.cuh"             // sampled_return, squashed_dim

using namespace wdb;

namespace {

bool make_plan(const wdb_ddpg_update_args *u, const wdb_replay_windows *w, Plan *p) {
  if (!u) return false;
  const wdb_ddpg_net *actors[2] = {&u->actor, &u->target_actor};
  const wdb_ddpg_net *critics[2] = {&u->critic, &u->target_critic};
  const wdb_ddpg_net *const *nets[2] = {actors, critics};
  const int count[2] = {2, 2};
  if (!plan_layout(u->n_envs, u->n_agents, u->obs_dim, u->action_dim, u->action_dim,
                   u->capacity, u->cursor, u->n_step, w, nets, count, p))
    return false;
  return plan_smem(p, 6 + 2 * (p->L[1] - 1) + (p->L[0] - 1),
                   2ll * (p->wfloats[0] + p->wfloats[1]), p->gfloats[0] + p->gfloats[1]);
}

// ---------------------------------------------------------------------------- loss rows
// Every pass kernel is a template over its row source, Windows:
//   NoWindows      every window of the ring: row g is logical window i = g / EN (slots from
//                  `cursor`) of agent row n = g % EN, and the last window bootstraps from slot
//                  C - 1 undiscounted (ddpg.py:62-79);
//   const int2 *   B sampled windows (wdb_replay_windows): row g = windows[g], M = B, and every
//                  window bootstraps discounted.
// The two differ only in where a row's step-0 and bootstrap slots are and in the n-step
// return; a kernel picks them with `if constexpr (kSampled)`.  The ring branches keep their
// statements in the order the pinned machine code (tests/test_td3_cpu.py) was compiled from:
// nvcc 12.9 allocates registers differently when they are reordered, so a value the code after
// a branch uses is declared before it and assigned inside, and nothing is hoisted out of it.
struct NoWindows {};

template <class Windows>
__global__ void __launch_bounds__(kThreads, 1)
ddpg_update_kernel(const __grid_constant__ wdb_ddpg_update_args U, const __grid_constant__ Plan Pg,
                   float *partials, double *psums, Windows windows) {
  constexpr bool kSampled = !std::is_same<Windows, NoWindows>::value;
  extern __shared__ __align__(16) float smem[];
  __shared__ Plan P;                           // dynamic indexing of the kernel parameter goes
  __shared__ double s_err[kRows], s_j[kRows];  // through local memory: copy it once
  if (threadIdx.x == 0) P = Pg;
  __syncthreads();
  const int tid = threadIdx.x;
  float *Wa = smem, *Wc = Wa + P.wfloats[0], *Wta = Wc + P.wfloats[1], *Wtc = Wta + P.wfloats[0];
  float *Ga = Wtc + P.wfloats[1], *Gc = Ga + P.gfloats[0];
  const int g_total = P.gfloats[0] + P.gfloats[1];
  float *XQ = Ga + ((g_total + 3) / 4) * 4;      // obs ++ actions
  float *XJ = XQ + kTile;                      // obs ++ pi (target path: scratch)
  float *V = XJ + kTile;                       // columns: 0 target Q, 1 Q, 2 J, 4 dQ, 8 dJ
  float *Z = V + kTile;                        // actor head pre-activation
  float *D0 = Z + kTile, *D1 = D0 + kTile;     // deltas (target path: obs' and scratch)
  float *HQ = D1 + kTile;                      // critic hidden outputs, (obs, actions) path
  float *HJ = HQ + (P.L[1] - 1) * kTile;       // critic hidden outputs, (obs, pi) path
  float *HA = HJ + (P.L[1] - 1) * kTile;       // actor hidden outputs

  load_net(Wa, U.actor, P, 0);
  load_net(Wc, U.critic, P, 1);
  load_net(Wta, U.target_actor, P, 0);
  load_net(Wtc, U.target_critic, P, 1);
  for (int e = tid; e < g_total; e += kThreads) Ga[e] = 0.0f;
  for (int e = tid; e < P.n_buf * kTile; e += kThreads) XQ[e] = 0.0f;
  __syncthreads();

  const int F = U.obs_dim, A = U.action_dim, FA = F + A;
  const int C = U.capacity, cursor = U.cursor, ns = U.n_step, valid = P.valid;
  const long long EN = P.EN, M = P.M, E = U.n_envs, Np = U.n_agents;
  const float gamma = U.gamma, scale = U.action_scale, bias = U.action_bias;
  const float norm_q = (float)(2.0 / (double)M);         // mse_loss backward: 2 / numel
  const float d_j = -1.0f / (float)M;                    // -mean backward
  auto phys = [&](int k) { const int s = cursor + k; return s >= C ? s - C : s; };
  auto target_slot = [&](int i) { return i < valid - 1 ? i + ns : C - 1; };
  double err_acc = 0.0, j_acc = 0.0;

  for (long long g0 = (long long)blockIdx.x * kRows; g0 < M; g0 += (long long)gridDim.x * kRows) {
    // ---- inputs: XQ = obs ++ actions at slot i, D0 = obs at the bootstrap slot
    for (int e = tid; e < kRows * FA; e += kThreads) {
      const int r = e / FA, c = e - r * FA;
      const long long g = g0 + r;
      float xq = 0.0f, xt = 0.0f;
      if (g < M) {
        if constexpr (kSampled) {
          const SampledRows rows = {windows, C};
          const Row w = rows.at(g);
          const long long row = (long long)rows.slot(w, 0) * EN + w.n;
          if (c < F) {
            xq = U.obs[row * F + c];
            xt = U.obs[((long long)rows.slot(w, ns) * EN + w.n) * F + c];
          } else {
            xq = U.actions[row * A + (c - F)];
          }
        } else {
          const int i = (int)(g / EN);
          const long long n = g - (long long)i * EN;
          const long long row = (long long)phys(i) * EN + n;
          if (c < F) {
            xq = U.obs[row * F + c];
            xt = U.obs[((long long)phys(target_slot(i)) * EN + n) * F + c];
          } else {
            xq = U.actions[row * A + (c - F)];
          }
        }
      }
      XQ[r * kPitch + c] = xq;
      if (c < F) D0[r * kPitch + c] = xt;
    }
    __syncthreads();
    // ---- target actor -> a' = scale * tanh(z) + bias into D0's action columns
    net_forward(Wta, P, 0, D0,
                [&](int l) { return l == P.L[0] - 1 ? Z : (l % 2 == 0 ? D1 : XJ); });
    for (int e = tid; e < kRows * A; e += kThreads) {
      const int r = e / A, c = e - r * A;
      D0[r * kPitch + F + c] = __fadd_rn(__fmul_rn(scale, tanhf(Z[r * kPitch + c])), bias);
    }
    __syncthreads();
    // ---- target critic -> V[., 0]; critic on (obs, actions) -> V[., 1]; actor -> Z
    net_forward(Wtc, P, 1, D0,
                [&](int l) { return l == P.L[1] - 1 ? V : (l % 2 == 0 ? D1 : XJ); });
    net_forward(Wc, P, 1, XQ,
                [&](int l) { return l == P.L[1] - 1 ? V + 1 : HQ + l * kTile; });
    net_forward(Wa, P, 0, XQ,
                [&](int l) { return l == P.L[0] - 1 ? Z : HA + l * kTile; });
    // ---- critic on (obs, pi) -> V[., 2]
    for (int e = tid; e < kRows * FA; e += kThreads) {
      const int r = e / FA, c = e - r * FA;
      XJ[r * kPitch + c] = c < F ? XQ[r * kPitch + c]
                                 : __fadd_rn(__fmul_rn(scale, tanhf(Z[r * kPitch + c - F])), bias);
    }
    __syncthreads();
    net_forward(Wc, P, 1, XJ,
                [&](int l) { return l == P.L[1] - 1 ? V + 2 : HJ + l * kTile; });
    // ---- n-step return (ddpg.py:62-79, same float32 operations) and the loss gradients
    if (tid < kRows) {
      const int r = tid;
      const long long g = g0 + r;
      float dq = 0.0f, dj = 0.0f;
      if (g < M) {
        float q, jv, ret;
        if constexpr (kSampled) {
          const SampledRows rows = {windows, C};
          const float qt = V[r * kPitch];
          q = V[r * kPitch + 1];
          jv = V[r * kPitch + 2];
          ret = sampled_return(U, P, rows, rows.at(g), qt);
        } else {
          const int i = (int)(g / EN);
          const long long n = g - (long long)i * EN, env = n / Np;
          const float qt = V[r * kPitch];
          q = V[r * kPitch + 1];
          jv = V[r * kPitch + 2];
          const int pl = phys(i + ns - 1);
          const float rl = U.rewards[(long long)pl * EN + n];
          const float dl = (float)U.done[(long long)pl * E + env];
          const float om = __fsub_rn(1.0f, dl);
          ret = i < valid - 1 ? __fadd_rn(rl, __fmul_rn(__fmul_rn(om, gamma), qt))
                              : __fadd_rn(__fmul_rn(dl, rl), __fmul_rn(om, qt));
          for (int j = 1; j < ns; j++) {
            const int pk = phys(ns - 1 - j + i);
            const float dk = (float)U.done[(long long)pk * E + env];
            ret = __fadd_rn(__fmul_rn(__fmul_rn(__fsub_rn(1.0f, dk), gamma), ret),
                            U.rewards[(long long)pk * EN + n]);
          }
        }
        const float diff = __fsub_rn(q, ret);
        dq = __fmul_rn(diff, norm_q);
        dj = d_j;
        err_acc += (double)diff * (double)diff;
        j_acc += (double)jv;
        if (U.values) U.values[g] = q;
        if (U.j_values) U.j_values[g] = jv;
        if (U.returns) U.returns[g] = ret;
      }
      V[r * kPitch + 4] = dq;
      V[r * kPitch + 8] = dj;
    }
    __syncthreads();
    // ---- backward: critic on both paths, then the tanh head and the actor
    net_backward(Wc, P, 1, Gc, V + 4,
                 [&](int l) { return l == 0 ? XQ : HQ + (l - 1) * kTile; }, D0, D1, -1);
    const float *dpi = net_backward(
        Wc, P, 1, Gc, V + 8, [&](int l) { return l == 0 ? XJ : HJ + (l - 1) * kTile; }, D0, D1, F);
    float *dz = dpi == D0 ? D1 : D0;
    for (int e = tid; e < kRows * A; e += kThreads) {
      const int r = e / A, c = e - r * A;
      const float y = tanhf(Z[r * kPitch + c]);
      dz[r * kPitch + c] = __fmul_rn(__fmul_rn(dpi[r * kPitch + F + c], scale),
                                     __fsub_rn(1.0f, __fmul_rn(y, y)));
    }
    __syncthreads();
    net_backward(Wa, P, 0, Ga, dz, [&](int l) { return l == 0 ? XQ : HA + (l - 1) * kTile; },
                 D0, D1, -1);
  }

  // ---- this CTA's partials
  float *part = partials + (long long)blockIdx.x * g_total;
  for (int e = tid; e < g_total; e += kThreads) part[e] = Ga[e];
  if (tid < kRows) {
    s_err[tid] = err_acc;
    s_j[tid] = j_acc;
  }
  __syncthreads();
  if (tid == 0) {
    double a = 0.0, b = 0.0;
    for (int r = 0; r < kRows; r++) {
      a += s_err[r];
      b += s_j[r];
    }
    psums[2 * blockIdx.x] = a;
    psums[2 * blockIdx.x + 1] = b;
  }
}

// ---------------------------------------------------------------------------- TD3
// The n-step return of loss row g (logical window i, agent row n) from the bootstrap value qt:
// ddpg.py:62-79's recursion in the same float32 operations as ddpg_update_kernel (TD3's and
// SAC's argument structs).
template <class Args>
__device__ __forceinline__ float td3_return(const Args &U, const Plan &P, int i, long long n,
                                            float qt) {
  const int C = U.capacity, ns = U.n_step;
  auto phys = [&](int k) { const int s = U.cursor + k; return s >= C ? s - C : s; };
  const long long EN = P.EN, E = U.n_envs, env = n / U.n_agents;
  const int pl = phys(i + ns - 1);
  const float rl = U.rewards[(long long)pl * EN + n];
  const float dl = (float)U.done[(long long)pl * E + env];
  const float om = __fsub_rn(1.0f, dl);
  float ret = i < P.valid - 1 ? __fadd_rn(rl, __fmul_rn(__fmul_rn(om, U.gamma), qt))
                              : __fadd_rn(__fmul_rn(dl, rl), __fmul_rn(om, qt));
  for (int j = 1; j < ns; j++) {
    const int pk = phys(ns - 1 - j + i);
    const float dk = (float)U.done[(long long)pk * E + env];
    ret = __fadd_rn(__fmul_rn(__fmul_rn(__fsub_rn(1.0f, dk), U.gamma), ret),
                    U.rewards[(long long)pk * EN + n]);
  }
  return ret;
}

// Critic pass: the gradients of mse(Q1, R) + mse(Q2, R) into per-CTA partials [G1 | G2].
template <class Windows>
__global__ void __launch_bounds__(kThreads, 1)
td3_critic_kernel(const __grid_constant__ wdb_td3_update_args U, const __grid_constant__ Plan Pg,
                  float *partials, double *psums, Windows windows) {
  constexpr bool kSampled = !std::is_same<Windows, NoWindows>::value;
  extern __shared__ __align__(16) float smem[];
  __shared__ Plan P;
  __shared__ double s_e1[kRows], s_e2[kRows];
  if (threadIdx.x == 0) P = Pg;
  __syncthreads();
  const int tid = threadIdx.x;
  float *Wta = smem, *Wc1 = Wta + P.wfloats[0], *Wc2 = Wc1 + P.wfloats[1];
  float *Wt1 = Wc2 + P.wfloats[1], *Wt2 = Wt1 + P.wfloats[1];
  float *G1 = Wt2 + P.wfloats[1], *G2 = G1 + P.gfloats[1];
  const int g_total = 2 * P.gfloats[1];
  float *XQ = G1 + ((g_total + 3) / 4) * 4;      // obs ++ actions
  float *XS = XQ + kTile;                      // scratch of the target forwards
  float *V = XS + kTile;                       // columns: 0 Q1', 1 Q2', 2 Q1, 3 Q2, 4 dQ1, 8 dQ2
  float *Z = V + kTile;                        // target actor head pre-activation
  float *D0 = Z + kTile, *D1 = D0 + kTile;     // deltas (target path: obs' ++ a' and scratch)
  float *H1 = D1 + kTile;                      // Q1 hidden outputs
  float *H2 = H1 + (P.L[1] - 1) * kTile;       // Q2 hidden outputs

  load_net(Wta, U.target_actor, P, 0);
  load_net(Wc1, U.critic, P, 1);
  load_net(Wc2, U.critic2, P, 1);
  load_net(Wt1, U.target_critic, P, 1);
  load_net(Wt2, U.target_critic2, P, 1);
  for (int e = tid; e < g_total; e += kThreads) G1[e] = 0.0f;
  for (int e = tid; e < P.n_buf * kTile; e += kThreads) XQ[e] = 0.0f;
  __syncthreads();

  const int F = U.obs_dim, A = U.action_dim, FA = F + A;
  const int C = U.capacity, cursor = U.cursor, ns = U.n_step, valid = P.valid;
  const long long EN = P.EN, M = P.M;
  const float scale = U.action_scale, bias = U.action_bias;
  const float sd = __fmul_rn(U.target_noise, scale), clip = __fmul_rn(U.target_noise_clip, scale);
  const float lo = __fsub_rn(bias, scale), hi = __fadd_rn(bias, scale);
  const float norm_q = (float)(2.0 / (double)M);
  auto phys = [&](int k) { const int s = cursor + k; return s >= C ? s - C : s; };
  auto target_slot = [&](int i) { return i < valid - 1 ? i + ns : C - 1; };
  double e1_acc = 0.0, e2_acc = 0.0;

  for (long long g0 = (long long)blockIdx.x * kRows; g0 < M; g0 += (long long)gridDim.x * kRows) {
    // ---- inputs: XQ = obs ++ actions at slot i, D0 = obs at the bootstrap slot
    for (int e = tid; e < kRows * FA; e += kThreads) {
      const int r = e / FA, c = e - r * FA;
      const long long g = g0 + r;
      float xq = 0.0f, xt = 0.0f;
      if (g < M) {
        if constexpr (kSampled) {
          const SampledRows rows = {windows, C};
          const Row w = rows.at(g);
          const long long row = (long long)rows.slot(w, 0) * EN + w.n;
          if (c < F) {
            xq = U.obs[row * F + c];
            xt = U.obs[((long long)rows.slot(w, ns) * EN + w.n) * F + c];
          } else {
            xq = U.actions[row * A + (c - F)];
          }
        } else {
          const int i = (int)(g / EN);
          const long long n = g - (long long)i * EN;
          const long long row = (long long)phys(i) * EN + n;
          if (c < F) {
            xq = U.obs[row * F + c];
            xt = U.obs[((long long)phys(target_slot(i)) * EN + n) * F + c];
          } else {
            xq = U.actions[row * A + (c - F)];
          }
        }
      }
      XQ[r * kPitch + c] = xq;
      if (c < F) D0[r * kPitch + c] = xt;
    }
    __syncthreads();
    // ---- target actor + clipped noise -> a' into D0's action columns
    net_forward(Wta, P, 0, D0,
                [&](int l) { return l == P.L[0] - 1 ? Z : (l % 2 == 0 ? D1 : XS); });
    for (int e = tid; e < kRows * A; e += kThreads) {
      const int r = e / A, c = e - r * A;
      const long long g = g0 + r;
      const float pi = __fadd_rn(__fmul_rn(scale, tanhf(Z[r * kPitch + c])), bias);
      const float eps = g < M ? U.noise[g * A + c] : 0.0f;
      const float nz = fminf(fmaxf(__fmul_rn(eps, sd), -clip), clip);
      D0[r * kPitch + F + c] = fminf(fmaxf(__fadd_rn(pi, nz), lo), hi);
    }
    __syncthreads();
    // ---- target critics -> V[., 0], V[., 1]; critics on (obs, actions) -> V[., 2], V[., 3]
    net_forward(Wt1, P, 1, D0,
                [&](int l) { return l == P.L[1] - 1 ? V : (l % 2 == 0 ? D1 : XS); });
    net_forward(Wt2, P, 1, D0,
                [&](int l) { return l == P.L[1] - 1 ? V + 1 : (l % 2 == 0 ? D1 : XS); });
    net_forward(Wc1, P, 1, XQ,
                [&](int l) { return l == P.L[1] - 1 ? V + 2 : H1 + l * kTile; });
    net_forward(Wc2, P, 1, XQ,
                [&](int l) { return l == P.L[1] - 1 ? V + 3 : H2 + l * kTile; });
    // ---- the n-step return from min(Q1', Q2') and the loss gradients
    if (tid < kRows) {
      const int r = tid;
      const long long g = g0 + r;
      float d1 = 0.0f, d2 = 0.0f;
      if (g < M) {
        float q1, q2, ret;
        if constexpr (kSampled) {
          const SampledRows rows = {windows, C};
          const float qt = fminf(V[r * kPitch], V[r * kPitch + 1]);
          q1 = V[r * kPitch + 2];
          q2 = V[r * kPitch + 3];
          ret = sampled_return(U, P, rows, rows.at(g), qt);
        } else {
          const int i = (int)(g / EN);
          const long long n = g - (long long)i * EN;
          const float qt = fminf(V[r * kPitch], V[r * kPitch + 1]);
          q1 = V[r * kPitch + 2];
          q2 = V[r * kPitch + 3];
          ret = td3_return(U, P, i, n, qt);
        }
        const float e1 = __fsub_rn(q1, ret), e2 = __fsub_rn(q2, ret);
        d1 = __fmul_rn(e1, norm_q);
        d2 = __fmul_rn(e2, norm_q);
        e1_acc += (double)e1 * (double)e1;
        e2_acc += (double)e2 * (double)e2;
        if (U.q1_values) U.q1_values[g] = q1;
        if (U.q2_values) U.q2_values[g] = q2;
        if (U.returns) U.returns[g] = ret;
      }
      V[r * kPitch + 4] = d1;
      V[r * kPitch + 8] = d2;
    }
    __syncthreads();
    // ---- backward: each critic on (obs, actions) into its own gradient block
    net_backward(Wc1, P, 1, G1, V + 4,
                 [&](int l) { return l == 0 ? XQ : H1 + (l - 1) * kTile; }, D0, D1, -1);
    net_backward(Wc2, P, 1, G2, V + 8,
                 [&](int l) { return l == 0 ? XQ : H2 + (l - 1) * kTile; }, D0, D1, -1);
  }

  float *part = partials + (long long)blockIdx.x * g_total;
  for (int e = tid; e < g_total; e += kThreads) part[e] = G1[e];
  if (tid < kRows) {
    s_e1[tid] = e1_acc;
    s_e2[tid] = e2_acc;
  }
  __syncthreads();
  if (tid == 0) {
    double a = 0.0, b = 0.0;
    for (int r = 0; r < kRows; r++) {
      a += s_e1[r];
      b += s_e2[r];
    }
    psums[2 * blockIdx.x] = a;
    psums[2 * blockIdx.x + 1] = b;
  }
}

// Actor pass: the gradient of -mean Q1(obs, actor(obs)) into per-CTA actor partials; the
// critic's weights only carry the gradient to its action inputs.
template <class Windows>
__global__ void __launch_bounds__(kThreads, 1)
td3_actor_kernel(const __grid_constant__ wdb_td3_update_args U, const __grid_constant__ Plan Pg,
                 float *partials, double *psums, Windows windows) {
  constexpr bool kSampled = !std::is_same<Windows, NoWindows>::value;
  extern __shared__ __align__(16) float smem[];
  __shared__ Plan P;
  __shared__ double s_j[kRows];
  if (threadIdx.x == 0) P = Pg;
  __syncthreads();
  const int tid = threadIdx.x;
  float *Wa = smem, *Wc = Wa + P.wfloats[0];
  float *Ga = Wc + P.wfloats[1];
  const int g_total = P.gfloats[0];
  float *XJ = Ga + ((g_total + 3) / 4) * 4;      // obs ++ pi
  float *V = XJ + kTile;                       // columns: 0 J, 8 dJ
  float *Z = V + kTile;                        // actor head pre-activation
  float *D0 = Z + kTile, *D1 = D0 + kTile;     // deltas
  float *HJ = D1 + kTile;                      // Q1 hidden outputs on (obs, pi)
  float *HA = HJ + (P.L[1] - 1) * kTile;       // actor hidden outputs

  load_net(Wa, U.actor, P, 0);
  load_net(Wc, U.critic, P, 1);
  for (int e = tid; e < g_total; e += kThreads) Ga[e] = 0.0f;
  for (int e = tid; e < P.n_buf * kTile; e += kThreads) XJ[e] = 0.0f;
  __syncthreads();

  const int F = U.obs_dim, A = U.action_dim;
  const int C = U.capacity, cursor = U.cursor;
  const long long EN = P.EN, M = P.M;
  const float scale = U.action_scale, bias = U.action_bias;
  const float d_j = -1.0f / (float)M;
  auto phys = [&](int k) { const int s = cursor + k; return s >= C ? s - C : s; };
  double j_acc = 0.0;

  for (long long g0 = (long long)blockIdx.x * kRows; g0 < M; g0 += (long long)gridDim.x * kRows) {
    for (int e = tid; e < kRows * F; e += kThreads) {
      const int r = e / F, c = e - r * F;
      const long long g = g0 + r;
      float x = 0.0f;
      if (g < M) {
        if constexpr (kSampled) {
          const SampledRows rows = {windows, C};
          const Row w = rows.at(g);
          x = U.obs[((long long)rows.slot(w, 0) * EN + w.n) * F + c];
        } else {
          const int i = (int)(g / EN);
          const long long n = g - (long long)i * EN;
          x = U.obs[((long long)phys(i) * EN + n) * F + c];
        }
      }
      XJ[r * kPitch + c] = x;
    }
    __syncthreads();
    // ---- actor -> pi into XJ's action columns; Q1 on (obs, pi) -> V[., 0]
    net_forward(Wa, P, 0, XJ, [&](int l) { return l == P.L[0] - 1 ? Z : HA + l * kTile; });
    for (int e = tid; e < kRows * A; e += kThreads) {
      const int r = e / A, c = e - r * A;
      XJ[r * kPitch + F + c] = __fadd_rn(__fmul_rn(scale, tanhf(Z[r * kPitch + c])), bias);
    }
    __syncthreads();
    net_forward(Wc, P, 1, XJ, [&](int l) { return l == P.L[1] - 1 ? V : HJ + l * kTile; });
    if (tid < kRows) {
      const int r = tid;
      const long long g = g0 + r;
      float dj = 0.0f;
      if (g < M) {
        const float jv = V[r * kPitch];
        dj = d_j;
        j_acc += (double)jv;
        if (U.j_values) U.j_values[g] = jv;
      }
      V[r * kPitch + 8] = dj;
    }
    __syncthreads();
    // ---- backward: Q1 to its action inputs, the tanh head, the actor
    const float *dpi = net_backward<false>(
        Wc, P, 1, nullptr, V + 8, [&](int l) { return l == 0 ? XJ : HJ + (l - 1) * kTile; },
        D0, D1, F);
    float *dz = dpi == D0 ? D1 : D0;
    for (int e = tid; e < kRows * A; e += kThreads) {
      const int r = e / A, c = e - r * A;
      const float y = tanhf(Z[r * kPitch + c]);
      dz[r * kPitch + c] = __fmul_rn(__fmul_rn(dpi[r * kPitch + F + c], scale),
                                     __fsub_rn(1.0f, __fmul_rn(y, y)));
    }
    __syncthreads();
    net_backward(Wa, P, 0, Ga, dz, [&](int l) { return l == 0 ? XJ : HA + (l - 1) * kTile; },
                 D0, D1, -1);
  }

  float *part = partials + (long long)blockIdx.x * g_total;
  for (int e = tid; e < g_total; e += kThreads) part[e] = Ga[e];
  if (tid < kRows) s_j[tid] = j_acc;
  __syncthreads();
  if (tid == 0) {
    double a = 0.0;
    for (int r = 0; r < kRows; r++) a += s_j[r];
    psums[2 * blockIdx.x] = a;
    psums[2 * blockIdx.x + 1] = 0.0;
  }
}

// ---------------------------------------------------------------------------- SAC
// Critic pass: the gradients of mse(Q1, R) + mse(Q2, R) into per-CTA partials [G1 | G2], R
// bootstrapped with min(Q1', Q2')(obs', a') - alpha log pi(a' | obs'), a' from the actor.
template <class Windows>
__global__ void __launch_bounds__(kThreads, 1)
sac_critic_kernel(const __grid_constant__ wdb_sac_update_args U, const __grid_constant__ Plan Pg,
                  float *partials, double *psums, Windows windows) {
  constexpr bool kSampled = !std::is_same<Windows, NoWindows>::value;
  extern __shared__ __align__(16) float smem[];
  __shared__ Plan P;
  __shared__ double s_e1[kRows], s_e2[kRows];
  if (threadIdx.x == 0) P = Pg;
  __syncthreads();
  const int tid = threadIdx.x;
  float *Wa = smem, *Wc1 = Wa + P.wfloats[0], *Wc2 = Wc1 + P.wfloats[1];
  float *Wt1 = Wc2 + P.wfloats[1], *Wt2 = Wt1 + P.wfloats[1];
  float *G1 = Wt2 + P.wfloats[1], *G2 = G1 + P.gfloats[1];
  const int g_total = 2 * P.gfloats[1];
  float *XQ = G1 + ((g_total + 3) / 4) * 4;      // obs ++ actions
  float *XS = XQ + kTile;                      // scratch of the bootstrap forwards
  float *V = XS + kTile;                       // columns: 0 Q1', 1 Q2', 2 Q1, 3 Q2, 4 dQ1, 8 dQ2
  float *Z = V + kTile;                        // actor head on obs'; then [0, A): log-prob terms
  float *D0 = Z + kTile, *D1 = D0 + kTile;     // deltas (bootstrap path: obs' ++ a' and scratch)
  float *H1 = D1 + kTile;                      // Q1 hidden outputs
  float *H2 = H1 + (P.L[1] - 1) * kTile;       // Q2 hidden outputs

  load_net(Wa, U.actor, P, 0);
  load_net(Wc1, U.critic, P, 1);
  load_net(Wc2, U.critic2, P, 1);
  load_net(Wt1, U.target_critic, P, 1);
  load_net(Wt2, U.target_critic2, P, 1);
  for (int e = tid; e < g_total; e += kThreads) G1[e] = 0.0f;
  for (int e = tid; e < P.n_buf * kTile; e += kThreads) XQ[e] = 0.0f;
  __syncthreads();

  const int F = U.obs_dim, A = U.action_dim, FA = F + A;
  const int C = U.capacity, cursor = U.cursor, ns = U.n_step, valid = P.valid;
  const long long EN = P.EN, M = P.M;
  const float scale = U.action_scale, bias = U.action_bias;
  const float lo = U.log_std_min, hi = U.log_std_max;
  const float alpha = expf(*U.log_alpha);
  const float norm_q = (float)(2.0 / (double)M);
  auto phys = [&](int k) { const int s = cursor + k; return s >= C ? s - C : s; };
  auto target_slot = [&](int i) { return i < valid - 1 ? i + ns : C - 1; };
  double e1_acc = 0.0, e2_acc = 0.0;

  for (long long g0 = (long long)blockIdx.x * kRows; g0 < M; g0 += (long long)gridDim.x * kRows) {
    // ---- inputs: XQ = obs ++ actions at slot i, D0 = obs at the bootstrap slot
    for (int e = tid; e < kRows * FA; e += kThreads) {
      const int r = e / FA, c = e - r * FA;
      const long long g = g0 + r;
      float xq = 0.0f, xt = 0.0f;
      if (g < M) {
        if constexpr (kSampled) {
          const SampledRows rows = {windows, C};
          const Row w = rows.at(g);
          const long long row = (long long)rows.slot(w, 0) * EN + w.n;
          if (c < F) {
            xq = U.obs[row * F + c];
            xt = U.obs[((long long)rows.slot(w, ns) * EN + w.n) * F + c];
          } else {
            xq = U.actions[row * A + (c - F)];
          }
        } else {
          const int i = (int)(g / EN);
          const long long n = g - (long long)i * EN;
          const long long row = (long long)phys(i) * EN + n;
          if (c < F) {
            xq = U.obs[row * F + c];
            xt = U.obs[((long long)phys(target_slot(i)) * EN + n) * F + c];
          } else {
            xq = U.actions[row * A + (c - F)];
          }
        }
      }
      XQ[r * kPitch + c] = xq;
      if (c < F) D0[r * kPitch + c] = xt;
    }
    __syncthreads();
    // ---- actor on obs' -> a' ~ pi(. | obs') into D0's action columns, log-prob terms into Z
    net_forward(Wa, P, 0, D0,
                [&](int l) { return l == P.L[0] - 1 ? Z : (l % 2 == 0 ? D1 : XS); });
    for (int e = tid; e < kRows * A; e += kThreads) {
      const int r = e / A, c = e - r * A;
      const long long g = g0 + r;
      const float eps = g < M ? U.critic_noise[g * A + c] : 0.0f;
      const SquashedDim s = squashed_dim(Z + r * kPitch, A, c, eps, lo, hi);
      D0[r * kPitch + F + c] = __fadd_rn(__fmul_rn(scale, s.y), bias);
      Z[r * kPitch + c] = s.term;
    }
    __syncthreads();
    // ---- target critics -> V[., 0], V[., 1]; critics on (obs, actions) -> V[., 2], V[., 3]
    net_forward(Wt1, P, 1, D0,
                [&](int l) { return l == P.L[1] - 1 ? V : (l % 2 == 0 ? D1 : XS); });
    net_forward(Wt2, P, 1, D0,
                [&](int l) { return l == P.L[1] - 1 ? V + 1 : (l % 2 == 0 ? D1 : XS); });
    net_forward(Wc1, P, 1, XQ,
                [&](int l) { return l == P.L[1] - 1 ? V + 2 : H1 + l * kTile; });
    net_forward(Wc2, P, 1, XQ,
                [&](int l) { return l == P.L[1] - 1 ? V + 3 : H2 + l * kTile; });
    // ---- the n-step return from min(Q1', Q2') - alpha log pi' and the loss gradients
    if (tid < kRows) {
      const int r = tid;
      const long long g = g0 + r;
      float d1 = 0.0f, d2 = 0.0f;
      if (g < M) {
        float q1, q2, ret;
        if constexpr (kSampled) {
          const SampledRows rows = {windows, C};
          float lp = 0.0f;
          for (int c = 0; c < A; c++) lp += Z[r * kPitch + c];
          const float qt = __fsub_rn(fminf(V[r * kPitch], V[r * kPitch + 1]), __fmul_rn(alpha, lp));
          q1 = V[r * kPitch + 2];
          q2 = V[r * kPitch + 3];
          ret = sampled_return(U, P, rows, rows.at(g), qt);
        } else {
          const int i = (int)(g / EN);
          const long long n = g - (long long)i * EN;
          float lp = 0.0f;
          for (int c = 0; c < A; c++) lp += Z[r * kPitch + c];
          const float qt = __fsub_rn(fminf(V[r * kPitch], V[r * kPitch + 1]), __fmul_rn(alpha, lp));
          q1 = V[r * kPitch + 2];
          q2 = V[r * kPitch + 3];
          ret = td3_return(U, P, i, n, qt);
        }
        const float e1 = __fsub_rn(q1, ret), e2 = __fsub_rn(q2, ret);
        d1 = __fmul_rn(e1, norm_q);
        d2 = __fmul_rn(e2, norm_q);
        e1_acc += (double)e1 * (double)e1;
        e2_acc += (double)e2 * (double)e2;
        if (U.q1_values) U.q1_values[g] = q1;
        if (U.q2_values) U.q2_values[g] = q2;
        if (U.returns) U.returns[g] = ret;
      }
      V[r * kPitch + 4] = d1;
      V[r * kPitch + 8] = d2;
    }
    __syncthreads();
    // ---- backward: each critic on (obs, actions) into its own gradient block
    net_backward(Wc1, P, 1, G1, V + 4,
                 [&](int l) { return l == 0 ? XQ : H1 + (l - 1) * kTile; }, D0, D1, -1);
    net_backward(Wc2, P, 1, G2, V + 8,
                 [&](int l) { return l == 0 ? XQ : H2 + (l - 1) * kTile; }, D0, D1, -1);
  }

  float *part = partials + (long long)blockIdx.x * g_total;
  for (int e = tid; e < g_total; e += kThreads) part[e] = G1[e];
  if (tid < kRows) {
    s_e1[tid] = e1_acc;
    s_e2[tid] = e2_acc;
  }
  __syncthreads();
  if (tid == 0) {
    double a = 0.0, b = 0.0;
    for (int r = 0; r < kRows; r++) {
      a += s_e1[r];
      b += s_e2[r];
    }
    psums[2 * blockIdx.x] = a;
    psums[2 * blockIdx.x + 1] = b;
  }
}

// Actor pass: the gradient of mean(alpha log pi(a | obs) - min(Q1, Q2)(obs, a)) into per-CTA
// actor partials.  Both critics run forward; the one the minimum picks (ties: Q1) carries the
// row's gradient to its action inputs (the other's row delta is 0), then through the tanh,
// the reparameterisation and the clamp into mu and the log-std.
template <class Windows>
__global__ void __launch_bounds__(kThreads, 1)
sac_actor_kernel(const __grid_constant__ wdb_sac_update_args U, const __grid_constant__ Plan Pg,
                 float *partials, double *psums, Windows windows) {
  constexpr bool kSampled = !std::is_same<Windows, NoWindows>::value;
  extern __shared__ __align__(16) float smem[];
  __shared__ Plan P;
  __shared__ double s_q[kRows], s_lp[kRows];
  if (threadIdx.x == 0) P = Pg;
  __syncthreads();
  const int tid = threadIdx.x;
  float *Wa = smem, *Wc1 = Wa + P.wfloats[0], *Wc2 = Wc1 + P.wfloats[1];
  float *Ga = Wc2 + P.wfloats[1];
  const int g_total = P.gfloats[0];
  float *XJ = Ga + ((g_total + 3) / 4) * 4;      // obs ++ a
  float *V = XJ + kTile;                       // columns: 0 Q1, 1 Q2, 8 dQ1, 12 dQ2
  float *Z = V + kTile;                        // actor head: mu ++ raw log-std
  float *D0 = Z + kTile, *D1 = D0 + kTile;     // deltas
  float *DA = D1 + kTile;                      // log-prob terms, then Q1's action gradient
  float *H1 = DA + kTile;                      // Q1 hidden outputs on (obs, a)
  float *H2 = H1 + (P.L[1] - 1) * kTile;       // Q2 hidden outputs on (obs, a)
  float *HA = H2 + (P.L[1] - 1) * kTile;       // actor hidden outputs

  load_net(Wa, U.actor, P, 0);
  load_net(Wc1, U.critic, P, 1);
  load_net(Wc2, U.critic2, P, 1);
  for (int e = tid; e < g_total; e += kThreads) Ga[e] = 0.0f;
  for (int e = tid; e < P.n_buf * kTile; e += kThreads) XJ[e] = 0.0f;
  __syncthreads();

  const int F = U.obs_dim, A = U.action_dim;
  const int C = U.capacity, cursor = U.cursor;
  const long long EN = P.EN, M = P.M;
  const float scale = U.action_scale, bias = U.action_bias;
  const float lo = U.log_std_min, hi = U.log_std_max;
  const float alpha = expf(*U.log_alpha);
  const float d_q = -1.0f / (float)M;                    // d loss / d min(Q1, Q2)
  const float d_lp = alpha / (float)M;                   // d loss / d log pi
  auto phys = [&](int k) { const int s = cursor + k; return s >= C ? s - C : s; };
  double q_acc = 0.0, lp_acc = 0.0;

  for (long long g0 = (long long)blockIdx.x * kRows; g0 < M; g0 += (long long)gridDim.x * kRows) {
    for (int e = tid; e < kRows * F; e += kThreads) {
      const int r = e / F, c = e - r * F;
      const long long g = g0 + r;
      float x = 0.0f;
      if (g < M) {
        if constexpr (kSampled) {
          const SampledRows rows = {windows, C};
          const Row w = rows.at(g);
          x = U.obs[((long long)rows.slot(w, 0) * EN + w.n) * F + c];
        } else {
          const int i = (int)(g / EN);
          const long long n = g - (long long)i * EN;
          x = U.obs[((long long)phys(i) * EN + n) * F + c];
        }
      }
      XJ[r * kPitch + c] = x;
    }
    __syncthreads();
    // ---- actor -> a into XJ's action columns (log-prob terms into DA); Q1, Q2 on (obs, a)
    net_forward(Wa, P, 0, XJ, [&](int l) { return l == P.L[0] - 1 ? Z : HA + l * kTile; });
    for (int e = tid; e < kRows * A; e += kThreads) {
      const int r = e / A, c = e - r * A;
      const long long g = g0 + r;
      const float eps = g < M ? U.actor_noise[g * A + c] : 0.0f;
      const SquashedDim s = squashed_dim(Z + r * kPitch, A, c, eps, lo, hi);
      XJ[r * kPitch + F + c] = __fadd_rn(__fmul_rn(scale, s.y), bias);
      DA[r * kPitch + c] = s.term;
    }
    __syncthreads();
    net_forward(Wc1, P, 1, XJ, [&](int l) { return l == P.L[1] - 1 ? V : H1 + l * kTile; });
    net_forward(Wc2, P, 1, XJ, [&](int l) { return l == P.L[1] - 1 ? V + 1 : H2 + l * kTile; });
    if (tid < kRows) {
      const int r = tid;
      const long long g = g0 + r;
      float d1 = 0.0f, d2 = 0.0f;
      if (g < M) {
        const float q1 = V[r * kPitch], q2 = V[r * kPitch + 1];
        const bool first = q1 <= q2;
        float lp = 0.0f;
        for (int c = 0; c < A; c++) lp += DA[r * kPitch + c];
        d1 = first ? d_q : 0.0f;
        d2 = first ? 0.0f : d_q;
        q_acc += (double)(first ? q1 : q2);
        lp_acc += (double)lp;
        if (U.log_probs) U.log_probs[g] = lp;
      }
      V[r * kPitch + 8] = d1;
      V[r * kPitch + 12] = d2;
    }
    __syncthreads();
    // ---- backward: Q1 to its action inputs (kept in DA), Q2 likewise
    const float *da1 = net_backward<false>(
        Wc1, P, 1, nullptr, V + 8, [&](int l) { return l == 0 ? XJ : H1 + (l - 1) * kTile; },
        D0, D1, F);
    for (int e = tid; e < kRows * A; e += kThreads) {
      const int r = e / A, c = e - r * A;
      DA[r * kPitch + c] = da1[r * kPitch + F + c];
    }
    __syncthreads();
    const float *da2 = net_backward<false>(
        Wc2, P, 1, nullptr, V + 12, [&](int l) { return l == 0 ? XJ : H2 + (l - 1) * kTile; },
        D0, D1, F);
    // ---- the tanh, the reparameterisation, the log-prob's own terms and the clamp
    float *dz = da2 == D0 ? D1 : D0;
    for (int e = tid; e < kRows * A; e += kThreads) {
      const int r = e / A, c = e - r * A;
      const long long g = g0 + r;
      float dmu = 0.0f, dls = 0.0f;
      if (g < M) {
        const float eps = U.actor_noise[g * A + c];
        const SquashedDim s = squashed_dim(Z + r * kPitch, A, c, eps, lo, hi);
        const float da = __fadd_rn(DA[r * kPitch + c], da2[r * kPitch + F + c]);
        const float du = fmaf(__fmul_rn(da, scale), __fsub_rn(1.0f, __fmul_rn(s.y, s.y)),
                              __fmul_rn(d_lp, 2.0f * s.y));
        dmu = du;
        dls = s.in_range ? fmaf(__fmul_rn(du, s.sigma), eps, -d_lp) : 0.0f;
      }
      dz[r * kPitch + c] = dmu;
      dz[r * kPitch + A + c] = dls;
    }
    __syncthreads();
    net_backward(Wa, P, 0, Ga, dz, [&](int l) { return l == 0 ? XJ : HA + (l - 1) * kTile; },
                 D0, D1, -1);
  }

  float *part = partials + (long long)blockIdx.x * g_total;
  for (int e = tid; e < g_total; e += kThreads) part[e] = Ga[e];
  if (tid < kRows) {
    s_q[tid] = q_acc;
    s_lp[tid] = lp_acc;
  }
  __syncthreads();
  if (tid == 0) {
    double a = 0.0, b = 0.0;
    for (int r = 0; r < kRows; r++) {
      a += s_q[r];
      b += s_lp[r];
    }
    psums[2 * blockIdx.x] = a;
    psums[2 * blockIdx.x + 1] = b;
  }
}

// ---------------------------------------------------------------------------- DQN
// dqn_tile_pass and qr_dqn_plan: wdb_dqn_pass.cuh
__global__ void __launch_bounds__(kThreads, 1)
dqn_pass_kernel(const __grid_constant__ wdb_dqn_update_args U, const __grid_constant__ Plan Pg,
                float *partials, double *psums, const int2 *windows) {
  dqn_tile_pass<false>(U, Pg, partials, psums, windows, nullptr);
}

__global__ void __launch_bounds__(kThreads, 1)
dqn_weighted_kernel(const __grid_constant__ wdb_dqn_update_args U, const __grid_constant__ Plan Pg,
                    float *partials, double *psums, const int2 *windows, const float *weights) {
  dqn_tile_pass<true>(U, Pg, partials, psums, windows, weights);
}

// ---------------------------------------------------------------------------- QR-DQN
// wdb_qr_dqn_update_sampled's tile kernel: DQN's networks and forwards with a head of A * N
// quantiles (column a * N + i: quantile i of action a).  Per row: a* the first argmax of the
// quantile sums of online(obs') (double_q) or target(obs'), the N targets T_j (DQN's n-step
// recursion on each target(obs')[a*, j]), and the quantile Huber gradient of each theta_i =
// online(obs)[a, i] in column a * N + i.  The row's 16 threads share its N x N pairs: thread k
// owns the quantiles i = k, k + 16, ... and sums over j in order, so no atomics and an update
// is bit-reproducible.  kWeighted: row g's gradient and loss are scaled by weights[g] with one
// multiply each, so unit weights change no bit.
template <bool kWeighted>
__device__ __forceinline__ void qr_dqn_tile_pass(const wdb_dqn_update_args &U, const Plan &Pg,
                                                 int nq, float *partials, double *psums,
                                                 const int2 *windows, const float *weights) {
  constexpr int kLanes = kThreads / kRows;     // threads per row
  extern __shared__ __align__(16) float smem[];
  __shared__ Plan P;
  __shared__ double s_h[kRows], s_q[kRows];
  if (threadIdx.x == 0) P = Pg;
  __syncthreads();
  const int tid = threadIdx.x;
  float *Wq = smem, *Wt = Wq + P.wfloats[0];
  float *G = Wt + P.wfloats[0];
  const int g_total = P.gfloats[0];
  float *X = G + ((g_total + 3) / 4) * 4;      // obs at slot(0)
  float *XB = X + kTile;                       // bootstrap obs at slot(n_step), then T_j
  float *QS = XB + kTile;                      // online quantiles at obs
  float *QT = QS + kTile;                      // target quantiles at obs'
  float *QD = QT + kTile;                      // online quantiles at obs' (double_q)
  float *DQ = QD + kTile;                      // head delta
  float *D0 = DQ + kTile, *D1 = D0 + kTile;    // deltas (the obs' forwards: scratch)
  float *H = D1 + kTile;                       // online hidden outputs on obs

  load_net(Wq, U.q, P, 0);
  load_net(Wt, U.target_q, P, 0);
  for (int e = tid; e < g_total; e += kThreads) G[e] = 0.0f;
  for (int e = tid; e < P.n_buf * kTile; e += kThreads) X[e] = 0.0f;
  __syncthreads();

  const int F = U.obs_dim, A = U.n_actions, N = nq, L = P.L[0], ns = U.n_step;
  const SampledRows rows = {windows, U.capacity};
  const long long EN = P.EN, M = P.M, E = U.n_envs, Np = U.n_agents;
  const float gamma = U.gamma, kappa = U.huber_delta;
  // d loss / d theta_i = -(1 / (kappa N B)) sum_j |tau_i - 1{u_ij < 0}| clamp(u_ij, -kappa, kappa)
  const float norm = (float)(1.0 / ((double)kappa * (double)N * (double)M));
  const int r = tid / kLanes, k = tid - r * kLanes;
  double h_acc = 0.0, q_acc = 0.0;

  for (long long g0 = (long long)blockIdx.x * kRows; g0 < M; g0 += (long long)gridDim.x * kRows) {
    // ---- inputs: X = obs at slot(0), XB = obs at slot(n_step)
    for (int e = tid; e < kRows * F; e += kThreads) {
      const int rr = e / F, c = e - rr * F;
      const long long g = g0 + rr;
      float x = 0.0f, xb = 0.0f;
      if (g < M) {
        const Row w = rows.at(g);
        x = U.obs[((long long)rows.slot(w, 0) * EN + w.n) * F + c];
        xb = U.obs[((long long)rows.slot(w, ns) * EN + w.n) * F + c];
      }
      X[rr * kPitch + c] = x;
      XB[rr * kPitch + c] = xb;
    }
    __syncthreads();
    net_forward(Wq, P, 0, X, [&](int l) { return l == L - 1 ? QS : H + l * kTile; });
    net_forward(Wt, P, 0, XB, [&](int l) { return l == L - 1 ? QT : (l % 2 == 0 ? D0 : D1); });
    if (U.double_q)
      net_forward(Wq, P, 0, XB, [&](int l) { return l == L - 1 ? QD : (l % 2 == 0 ? D0 : D1); });
    // ---- per row (its kLanes threads): a*, the targets T_j into XB, a zeroed head delta
    const long long g = g0 + r;
    float *dq = DQ + r * kPitch, *T = XB + r * kPitch;
    for (int c = k; c < A * N; c += kLanes) dq[c] = 0.0f;
    Row w = {0, 0};
    int a = -1;
    if (g < M) {
      w = rows.at(g);
      a = U.actions[(long long)rows.slot(w, 0) * EN + w.n];
      const float *qa = U.double_q ? QD + r * kPitch : QT + r * kPitch;
      int best = 0;                            // the first maximum of the quantile sums
      float best_sum = 0.0f;
      for (int c = 0; c < A; c++) {
        float s = 0.0f;
        for (int j = 0; j < N; j++) s = __fadd_rn(s, qa[c * N + j]);
        if (c == 0 || best_sum < s) { best_sum = s; best = c; }
      }
      const float *boot = QT + r * kPitch + best * N;
      const long long env = w.n / Np;
      for (int j = k; j < N; j += kLanes) {
        float ret = boot[j];
        for (int t = ns - 1; t >= 0; t--) {
          const int pk = rows.slot(w, t);
          const float om = U.done[(long long)pk * E + env] != 0 ? 0.0f : 1.0f;
          ret = __fadd_rn(__fmul_rn(__fmul_rn(om, gamma), ret),
                          U.rewards[(long long)pk * EN + w.n]);
        }
        T[j] = ret;
      }
    }
    __syncthreads();
    // ---- the pairs: thread k, quantiles i = k, k + kLanes, ...; T_j in order
    // (an action outside [0, A) -- never written by the samplers -- contributes nothing)
    if (g < M && a >= 0 && a < A) {
      const float *theta = QS + r * kPitch + a * N;
      const float wg = kWeighted ? weights[g] : 1.0f;
      double h_row = 0.0;
      for (int i = k; i < N; i += kLanes) {
        const float th = theta[i];
        const float tau = (float)(2 * i + 1) / (float)(2 * N);
        float acc = 0.0f;
        for (int j = 0; j < N; j++) {
          const float u = __fsub_rn(T[j], th);
          const float m = u < 0.0f ? __fsub_rn(1.0f, tau) : tau;     // |tau - 1{u < 0}|
          acc = fmaf(m, fminf(fmaxf(u, -kappa), kappa), acc);
          const double au = fabs((double)u);
          h_row += (double)m * (au < (double)kappa ? 0.5 * au * au
                                                   : (double)kappa * (au - 0.5 * (double)kappa));
        }
        if constexpr (kWeighted) acc = __fmul_rn(acc, wg);
        dq[a * N + i] = __fmul_rn(-acc, norm);
      }
      if constexpr (kWeighted) h_row *= (double)wg;
      h_acc += h_row;
    }
    if (k == 0 && g < M) {                     // the row's mean quantile and mean target
      double rbar = 0.0;
      for (int j = 0; j < N; j++) rbar += (double)T[j];
      rbar /= (double)N;
      if (U.returns) U.returns[g] = (float)rbar;
      if (a >= 0 && a < A) {
        double qbar = 0.0;
        for (int i = 0; i < N; i++) qbar += (double)QS[r * kPitch + a * N + i];
        qbar /= (double)N;
        q_acc += qbar;
        if (U.q_values) U.q_values[g] = (float)qbar;
      }
    }
    __syncthreads();
    net_backward(Wq, P, 0, G, DQ, [&](int l) { return l == 0 ? X : H + (l - 1) * kTile; }, D0,
                 D1, -1);
  }

  // ---- this CTA's partials: sums[0] = sum_g w_g loss_g, sums[1] = sum_g mean_i theta_i
  float *part = partials + (long long)blockIdx.x * g_total;
  for (int e = tid; e < g_total; e += kThreads) part[e] = G[e];
  for (int off = kLanes / 2; off > 0; off /= 2)   // the row's lanes, in a fixed order
    h_acc += __shfl_xor_sync(0xffffffffu, h_acc, off, kLanes);
  if (k == 0) {
    s_h[r] = h_acc;
    s_q[r] = q_acc;
  }
  __syncthreads();
  if (tid == 0) {
    double a = 0.0, b = 0.0;
    for (int t = 0; t < kRows; t++) {
      a += s_h[t];
      b += s_q[t];
    }
    psums[2 * blockIdx.x] = a / ((double)kappa * (double)N);
    psums[2 * blockIdx.x + 1] = b;
  }
}

__global__ void __launch_bounds__(kThreads, 1)
qr_dqn_kernel(const __grid_constant__ wdb_dqn_update_args U, const __grid_constant__ Plan Pg,
              int nq, float *partials, double *psums, const int2 *windows) {
  qr_dqn_tile_pass<false>(U, Pg, nq, partials, psums, windows, nullptr);
}

__global__ void __launch_bounds__(kThreads, 1)
qr_dqn_prioritized_kernel(const __grid_constant__ wdb_dqn_update_args U,
                          const __grid_constant__ Plan Pg, int nq, float *partials,
                          double *psums, const int2 *windows, const float *weights) {
  qr_dqn_tile_pass<true>(U, Pg, nq, partials, psums, windows, weights);
}

// ---------------------------------------------------------------------------- host side
// TD3's plan of one pass: the actor shape (actor, target actor) and the critic shape (both
// critics and their targets) as in DDPG; the critic pass holds the target actor, four critics
// and both critic gradient blocks, the actor pass the actor, Q1 and the actor gradients.
bool td3_plan(const wdb_td3_update_args *u, const wdb_replay_windows *w, bool actor_pass,
              Plan *p) {
  if (!u) return false;
  if (!(u->target_noise >= 0.0f) || !(u->target_noise_clip >= 0.0f)) return false;
  const wdb_ddpg_net *actors[2] = {&u->actor, &u->target_actor};
  const wdb_ddpg_net *critics[4] = {&u->critic, &u->critic2, &u->target_critic,
                                    &u->target_critic2};
  const wdb_ddpg_net *const *nets[2] = {actors, critics};
  const int count[2] = {2, 4};
  if (!plan_layout(u->n_envs, u->n_agents, u->obs_dim, u->action_dim, u->action_dim,
                   u->capacity, u->cursor, u->n_step, w, nets, count, p))
    return false;
  if (actor_pass)
    return plan_smem(p, 5 + (p->L[1] - 1) + (p->L[0] - 1), p->wfloats[0] + p->wfloats[1],
                     p->gfloats[0]);
  return plan_smem(p, 6 + 2 * (p->L[1] - 1), p->wfloats[0] + 4ll * p->wfloats[1],
                   2 * p->gfloats[1]);
}

long long td3_workspace_bytes(const Plan &P, bool actor_pass) {
  return 16ll * P.grid + 4ll * P.grid * (actor_pass ? P.gfloats[0] : 2 * P.gfloats[1]);
}

bool nets_ok(const wdb_ddpg_update_args *u, const Plan &P) {
  const wdb_ddpg_net *nets[4] = {&u->actor, &u->critic, &u->target_actor, &u->target_critic};
  for (int k = 0; k < 4; k++)
    for (int l = 0; l < P.L[k % 2]; l++) {
      if (!nets[k]->w[l] || !nets[k]->b[l]) return false;
      if (k < 2 && (!nets[k]->gw[l] || !nets[k]->gb[l])) return false;
    }
  return true;
}

// SAC's plan of one pass: the actor shape (head 2A) and the critic shape (both critics and
// their targets); the critic pass holds the actor, four critics and both critic gradient
// blocks, the actor pass the actor, both critics and the actor gradients.
bool sac_plan(const wdb_sac_update_args *u, const wdb_replay_windows *w, bool actor_pass,
              Plan *p) {
  if (!u) return false;
  if (!(u->log_std_min <= u->log_std_max)) return false;
  const wdb_ddpg_net *actors[1] = {&u->actor};
  const wdb_ddpg_net *critics[4] = {&u->critic, &u->critic2, &u->target_critic,
                                    &u->target_critic2};
  const wdb_ddpg_net *const *nets[2] = {actors, critics};
  const int count[2] = {1, 4};
  if (!plan_layout(u->n_envs, u->n_agents, u->obs_dim, u->action_dim, 2 * u->action_dim,
                   u->capacity, u->cursor, u->n_step, w, nets, count, p))
    return false;
  if (actor_pass)
    return plan_smem(p, 6 + 2 * (p->L[1] - 1) + (p->L[0] - 1),
                     p->wfloats[0] + 2ll * p->wfloats[1], p->gfloats[0]);
  return plan_smem(p, 6 + 2 * (p->L[1] - 1), p->wfloats[0] + 4ll * p->wfloats[1],
                   2 * p->gfloats[1]);
}


// Launches one pass kernel (its NoWindows instantiation over every window of the ring, or its
// const int2 * one over w's windows) and the reduction R of its per-CTA partials into the
// gradient arena and `sums`.
template <class Args>
int launch_pass(void *stream, const Args *u, const Plan &P, const wdb_replay_windows *w,
                void (*ring)(const Args, const Plan, float *, double *, NoWindows),
                void (*sampled)(const Args, const Plan, float *, double *, const int2 *),
                size_t *configured, Reduce *R, int widest, double *sums) {
  if (!u->workspace || (w && !w->windows)) return (int)cudaErrorInvalidValue;
  const size_t smem = (size_t)P.smem_floats * sizeof(float);
  int rc = allow_smem(w ? (const void *)sampled : (const void *)ring, smem,
                      &configured[w ? 1 : 0]);
  if (rc != cudaSuccess) return rc;
  double *psums = static_cast<double *>(u->workspace);
  float *partials = reinterpret_cast<float *>(psums + 2 * P.grid);
  if (w)
    sampled<<<P.grid, kThreads, smem, as_stream(stream)>>>(
        *u, P, partials, psums, reinterpret_cast<const int2 *>(w->windows));
  else
    ring<<<P.grid, kThreads, smem, as_stream(stream)>>>(*u, P, partials, psums, NoWindows{});
  rc = finish_launch();
  if (rc != cudaSuccess) return rc;
  R->grid = P.grid;
  return launch_reduce(stream, *R, widest, partials, psums, sums);
}

int ddpg_update(void *stream, const wdb_ddpg_update_args *u, const wdb_replay_windows *w) {
  Plan P;
  if (!make_plan(u, w, &P) || !nets_ok(u, P)) return (int)cudaErrorInvalidValue;
  if (!u->obs || !u->actions || !u->rewards || !u->done) return (int)cudaErrorInvalidValue;
  Reduce R = {};
  R.g_total = P.gfloats[0] + P.gfloats[1];
  int widest = 1;
  add_segments(&R, P, 0, 0, u->actor, &widest);
  add_segments(&R, P, 1, P.gfloats[0], u->critic, &widest);
  static size_t configured[2] = {0, 0};
  return launch_pass(stream, u, P, w, ddpg_update_kernel<NoWindows>,
                     ddpg_update_kernel<const int2 *>, configured, &R, widest, u->sums);
}

int td3_critic_update(void *stream, const wdb_td3_update_args *u, const wdb_replay_windows *w) {
  Plan P;
  if (!td3_plan(u, w, false, &P)) return (int)cudaErrorInvalidValue;
  if (!net_ok(u->target_actor, P.L[0], false) || !net_ok(u->critic, P.L[1], true) ||
      !net_ok(u->critic2, P.L[1], true) || !net_ok(u->target_critic, P.L[1], false) ||
      !net_ok(u->target_critic2, P.L[1], false))
    return (int)cudaErrorInvalidValue;
  if (!u->obs || !u->actions || !u->rewards || !u->done || !u->noise)
    return (int)cudaErrorInvalidValue;
  Reduce R = {};
  R.g_total = 2 * P.gfloats[1];
  int widest = 1;
  add_segments(&R, P, 1, 0, u->critic, &widest);
  add_segments(&R, P, 1, P.gfloats[1], u->critic2, &widest);
  static size_t configured[2] = {0, 0};
  return launch_pass(stream, u, P, w, td3_critic_kernel<NoWindows>,
                     td3_critic_kernel<const int2 *>, configured, &R, widest, u->sums);
}

int td3_actor_update(void *stream, const wdb_td3_update_args *u, const wdb_replay_windows *w) {
  Plan P;
  if (!td3_plan(u, w, true, &P)) return (int)cudaErrorInvalidValue;
  if (!net_ok(u->actor, P.L[0], true) || !net_ok(u->critic, P.L[1], false))
    return (int)cudaErrorInvalidValue;
  if (!u->obs) return (int)cudaErrorInvalidValue;
  Reduce R = {};
  R.g_total = P.gfloats[0];
  int widest = 1;
  add_segments(&R, P, 0, 0, u->actor, &widest);
  static size_t configured[2] = {0, 0};
  return launch_pass(stream, u, P, w, td3_actor_kernel<NoWindows>,
                     td3_actor_kernel<const int2 *>, configured, &R, widest,
                     u->sums ? u->sums + 2 : nullptr);
}

int sac_critic_update(void *stream, const wdb_sac_update_args *u, const wdb_replay_windows *w) {
  Plan P;
  if (!sac_plan(u, w, false, &P)) return (int)cudaErrorInvalidValue;
  if (!net_ok(u->actor, P.L[0], false) || !net_ok(u->critic, P.L[1], true) ||
      !net_ok(u->critic2, P.L[1], true) || !net_ok(u->target_critic, P.L[1], false) ||
      !net_ok(u->target_critic2, P.L[1], false))
    return (int)cudaErrorInvalidValue;
  if (!u->obs || !u->actions || !u->rewards || !u->done || !u->critic_noise || !u->log_alpha)
    return (int)cudaErrorInvalidValue;
  Reduce R = {};
  R.g_total = 2 * P.gfloats[1];
  int widest = 1;
  add_segments(&R, P, 1, 0, u->critic, &widest);
  add_segments(&R, P, 1, P.gfloats[1], u->critic2, &widest);
  static size_t configured[2] = {0, 0};
  return launch_pass(stream, u, P, w, sac_critic_kernel<NoWindows>,
                     sac_critic_kernel<const int2 *>, configured, &R, widest, u->sums);
}

int sac_actor_update(void *stream, const wdb_sac_update_args *u, const wdb_replay_windows *w) {
  Plan P;
  if (!sac_plan(u, w, true, &P)) return (int)cudaErrorInvalidValue;
  if (!net_ok(u->actor, P.L[0], true) || !net_ok(u->critic, P.L[1], false) ||
      !net_ok(u->critic2, P.L[1], false))
    return (int)cudaErrorInvalidValue;
  if (!u->obs || !u->actor_noise || !u->log_alpha) return (int)cudaErrorInvalidValue;
  Reduce R = {};
  R.g_total = P.gfloats[0];
  int widest = 1;
  add_segments(&R, P, 0, 0, u->actor, &widest);
  static size_t configured[2] = {0, 0};
  return launch_pass(stream, u, P, w, sac_actor_kernel<NoWindows>,
                     sac_actor_kernel<const int2 *>, configured, &R, widest,
                     u->sums ? u->sums + 2 : nullptr);
}

// weights NULL: wdb_dqn_update_sampled; else wdb_dqn_update_prioritized.
int dqn_update_sampled(void *stream, const wdb_dqn_update_args *u, const wdb_replay_windows *w,
                       const float *weights) {
  Plan P;
  if (!qr_dqn_plan(u, 1, w, &P)) return (int)cudaErrorInvalidValue;
  static size_t configured[2] = {0, 0};
  return launch_q_pass(stream, u, P, w, weights, configured, nullptr, dqn_pass_kernel,
                       dqn_weighted_kernel, *u, P);
}

// weights NULL: the uniform-replay kernel; else the importance-weighted one.
int qr_dqn_update_sampled(void *stream, const wdb_dqn_update_args *u, int nq,
                          const wdb_replay_windows *w, const float *weights) {
  Plan P;
  if (!qr_dqn_plan(u, nq, w, &P)) return (int)cudaErrorInvalidValue;
  static size_t configured[2] = {0, 0};
  return launch_q_pass(stream, u, P, w, weights, configured, nullptr, qr_dqn_kernel,
                       qr_dqn_prioritized_kernel, *u, P, nq);
}

}  // namespace

// ---------------------------------------------------------------------------- entry points
// Each pass has a ring form and a _sampled form; the latter's _supported / _workspace_bytes
// take the number of windows B.
#define WDB_PASS_API(name, Args, plan, bytes)                                                  \
  WDB_API int wdb_##name##_supported(const Args *u) {                                          \
    Plan P;                                                                                    \
    return plan(u, nullptr, &P) ? 1 : 0;                                                       \
  }                                                                                            \
  WDB_API long long wdb_##name##_workspace_bytes(const Args *u) {                              \
    Plan P;                                                                                    \
    return plan(u, nullptr, &P) ? bytes(P) : -1;                                               \
  }                                                                                            \
  WDB_API int wdb_##name(void *stream, const Args *u) { return name(stream, u, nullptr); }     \
  WDB_API int wdb_##name##_sampled_supported(const Args *u, int n_windows) {                   \
    const wdb_replay_windows w = {nullptr, n_windows};                                         \
    Plan P;                                                                                    \
    return plan(u, &w, &P) ? 1 : 0;                                                            \
  }                                                                                            \
  WDB_API long long wdb_##name##_sampled_workspace_bytes(const Args *u, int n_windows) {       \
    const wdb_replay_windows w = {nullptr, n_windows};                                         \
    Plan P;                                                                                    \
    return plan(u, &w, &P) ? bytes(P) : -1;                                                    \
  }                                                                                            \
  WDB_API int wdb_##name##_sampled(void *stream, const Args *u, const wdb_replay_windows *w) { \
    return w ? name(stream, u, w) : (int)cudaErrorInvalidValue;                                \
  }

namespace {
bool td3_critic_plan(const wdb_td3_update_args *u, const wdb_replay_windows *w, Plan *p) {
  return td3_plan(u, w, false, p);
}
bool td3_actor_plan(const wdb_td3_update_args *u, const wdb_replay_windows *w, Plan *p) {
  return td3_plan(u, w, true, p);
}
bool sac_critic_plan(const wdb_sac_update_args *u, const wdb_replay_windows *w, Plan *p) {
  return sac_plan(u, w, false, p);
}
bool sac_actor_plan(const wdb_sac_update_args *u, const wdb_replay_windows *w, Plan *p) {
  return sac_plan(u, w, true, p);
}
long long critic_bytes(const Plan &P) { return td3_workspace_bytes(P, false); }
long long actor_bytes(const Plan &P) { return td3_workspace_bytes(P, true); }
}  // namespace

WDB_PASS_API(ddpg_update, wdb_ddpg_update_args, make_plan, workspace_bytes)
WDB_PASS_API(td3_critic_update, wdb_td3_update_args, td3_critic_plan, critic_bytes)
WDB_PASS_API(td3_actor_update, wdb_td3_update_args, td3_actor_plan, actor_bytes)
WDB_PASS_API(sac_critic_update, wdb_sac_update_args, sac_critic_plan, critic_bytes)
WDB_PASS_API(sac_actor_update, wdb_sac_update_args, sac_actor_plan, actor_bytes)

// DQN has the sampled form only (it always trains from the replay buffer)
WDB_API int wdb_dqn_update_sampled_supported(const wdb_dqn_update_args *u, int n_windows) {
  const wdb_replay_windows w = {nullptr, n_windows};
  Plan P;
  return qr_dqn_plan(u, 1, &w, &P) ? 1 : 0;
}
WDB_API long long wdb_dqn_update_sampled_workspace_bytes(const wdb_dqn_update_args *u,
                                                         int n_windows) {
  const wdb_replay_windows w = {nullptr, n_windows};
  Plan P;
  return qr_dqn_plan(u, 1, &w, &P) ? dqn_workspace_bytes(P) : -1;
}
WDB_API int wdb_dqn_update_sampled(void *stream, const wdb_dqn_update_args *u,
                                   const wdb_replay_windows *w) {
  return dqn_update_sampled(stream, u, w, nullptr);
}

// The importance-weighted pass has the unweighted one's shapes and workspace
WDB_API int wdb_dqn_update_prioritized_supported(const wdb_dqn_update_args *u, int n_windows) {
  return wdb_dqn_update_sampled_supported(u, n_windows);
}
WDB_API long long wdb_dqn_update_prioritized_workspace_bytes(const wdb_dqn_update_args *u,
                                                             int n_windows) {
  return wdb_dqn_update_sampled_workspace_bytes(u, n_windows);
}
WDB_API int wdb_dqn_update_prioritized(void *stream, const wdb_dqn_update_args *u,
                                       const wdb_replay_windows *w, const float *weights) {
  return weights ? dqn_update_sampled(stream, u, w, weights) : (int)cudaErrorInvalidValue;
}

// QR-DQN: DQN's argument struct, plus the number of quantiles per action
WDB_API int wdb_qr_dqn_update_sampled_supported(const wdb_dqn_update_args *u, int n_quantiles,
                                                int n_windows) {
  const wdb_replay_windows w = {nullptr, n_windows};
  Plan P;
  return qr_dqn_plan(u, n_quantiles, &w, &P) ? 1 : 0;
}
WDB_API long long wdb_qr_dqn_update_sampled_workspace_bytes(const wdb_dqn_update_args *u,
                                                            int n_quantiles, int n_windows) {
  const wdb_replay_windows w = {nullptr, n_windows};
  Plan P;
  return qr_dqn_plan(u, n_quantiles, &w, &P) ? dqn_workspace_bytes(P) : -1;
}
WDB_API int wdb_qr_dqn_update_sampled(void *stream, const wdb_dqn_update_args *u,
                                      int n_quantiles, const wdb_replay_windows *w,
                                      const float *weights) {
  return qr_dqn_update_sampled(stream, u, n_quantiles, w, weights);
}
