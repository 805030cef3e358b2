// wdb_sac_discrete.cu -- one discrete-action SAC update (Christodoulou 2019, "Soft Actor-Critic
// for Discrete Action Settings") of one policy over B sampled replay windows, as two passes of
// two launches each: a tile kernel and the fixed-order reduction of its per-CTA partials
// (include/wdb200.h, wdb_sac_discrete_{critic,actor}_update_sampled).
//
// The actor and the four Q networks all map F -> A: the actor's head is A logits (a softmax
// policy), each Q network's head A action values.  Because the policy is categorical, every
// expectation over actions is exact: no reparameterisation noise, no tanh Jacobian.
//   critic pass, per tile of kRows windows: the actor, Q1' and Q2' on obs' (slot n_step), Q1 and
//     Q2 on obs (slot 0, their hidden outputs kept); per row, on the row's own thread, the
//     log-softmax of the logits, V' = sum_a pi'_a (min(Q1', Q2')_a - alpha log pi'_a), DQN's
//     n-step return R from V' (every non-zero done flag terminal), and dQk = 2 (Qk[a] - R) / B
//     in column a of each critic's head delta; then back through each critic into its own block.
//   actor pass, per tile: the actor (hidden outputs kept), Q1 and Q2 on obs; per row the
//     log-softmax, h_a = alpha log pi_a - min(Q1, Q2)_a and the logit delta
//     pi_j (h_j - sum_a pi_a h_a) / B; then back through the actor.
// Every sum over actions runs a = 0 .. A - 1 in order, and the partials are reduced in CTA order
// with no float atomics: a relaunch is bit-identical.  alpha = expf(*log_alpha) is read on the
// device.  Its own translation unit, on the primitives of wdb_update_tiles.cuh, so every other
// update kernel keeps its machine code.
#include "wdb_common.cuh"
#include "wdb_update_tiles.cuh"

using namespace wdb;

namespace {

// The plan of one pass.  plan_layout lays out an F -> head slot and an F + A -> 1 slot, so it is
// called twice with an action width of 1 for the unused critic-shaped slot (as qr_dqn_plan
// does): the actor in slot 0, then the four Q networks in slot 0 of a second plan, whose slot-0
// layout is copied into slot 1.  The layer steps index only P.*[k][l], so slot 1 then runs as an
// F -> A network.  The critic pass holds the actor, four Q networks, both critic gradient blocks
// and 9 + 2 (hidden layers) row tiles; the actor pass the actor, Q1, Q2, the actor gradient block
// and 6 + (actor hidden layers) row tiles.
bool sac_discrete_plan(const wdb_sac_discrete_update_args *u, const wdb_replay_windows *w,
                       bool actor_pass, Plan *p) {
  if (!u || !w) return false;
  const int A = u->n_actions;
  if (A < 2 || A > kMaxWidth) return false;
  const wdb_ddpg_net *actor[1] = {&u->actor};
  const wdb_ddpg_net *qs[4] = {&u->critic, &u->critic2, &u->target_critic, &u->target_critic2};
  const wdb_ddpg_net *const *actor_nets[2] = {actor, actor};
  const wdb_ddpg_net *const *q_nets[2] = {qs, qs};
  const int actor_count[2] = {1, 1}, q_count[2] = {4, 4};
  Plan q;
  if (!plan_layout(u->n_envs, u->n_agents, u->obs_dim, 1, A, u->capacity, 0, u->n_step, w,
                   actor_nets, actor_count, p) ||
      !plan_layout(u->n_envs, u->n_agents, u->obs_dim, 1, A, u->capacity, 0, u->n_step, w, q_nets,
                   q_count, &q))
    return false;
  p->L[1] = q.L[0];
  for (int l = 0; l < 4; l++) {
    p->in[1][l] = q.in[0][l];
    p->out[1][l] = q.out[0][l];
    p->pw[1][l] = q.pw[0][l];
    p->woff[1][l] = q.woff[0][l];
    p->goff[1][l] = q.goff[0][l];
  }
  p->wfloats[1] = q.wfloats[0];
  p->gfloats[1] = q.gfloats[0];
  if (actor_pass)
    return plan_smem(p, 6 + (p->L[0] - 1), p->wfloats[0] + 2ll * p->wfloats[1], p->gfloats[0]);
  return plan_smem(p, 9 + 2 * (p->L[1] - 1), p->wfloats[0] + 4ll * p->wfloats[1],
                   2 * p->gfloats[1]);
}

long long sac_discrete_workspace_bytes(const Plan &P, bool actor_pass) {
  return 16ll * P.grid + 4ll * P.grid * (actor_pass ? P.gfloats[0] : 2 * P.gfloats[1]);
}

// Writes this CTA's gradient block and its two double sums (the kRows row threads' in order).
__device__ __forceinline__ void write_partials(const float *G, int g_total, double a_acc,
                                               double b_acc, double *s_a, double *s_b,
                                               float *partials, double *psums) {
  const int tid = threadIdx.x;
  float *part = partials + (long long)blockIdx.x * g_total;
  for (int e = tid; e < g_total; e += kThreads) part[e] = G[e];
  if (tid < kRows) {
    s_a[tid] = a_acc;
    s_b[tid] = b_acc;
  }
  __syncthreads();
  if (tid == 0) {
    double a = 0.0, b = 0.0;
    for (int r = 0; r < kRows; r++) {
      a += s_a[r];
      b += s_b[r];
    }
    psums[2 * blockIdx.x] = a;
    psums[2 * blockIdx.x + 1] = b;
  }
}

// Critic pass: the gradients of mse(Q1(obs)[a], R) + mse(Q2(obs)[a], R) into per-CTA partials
// [G1 | G2]; psums: sum (Q1 - R)^2, sum (Q2 - R)^2.
__global__ void __launch_bounds__(kThreads, 1)
sac_discrete_critic_kernel(const __grid_constant__ wdb_sac_discrete_update_args U,
                           const __grid_constant__ Plan Pg, float *partials, double *psums,
                           const int2 *windows) {
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
  float *X = G1 + ((g_total + 3) / 4) * 4;     // obs at slot(0)
  float *XB = X + kTile;                       // obs' at slot(n_step)
  float *Z = XB + kTile;                       // actor logits on obs'
  float *QT1 = Z + kTile, *QT2 = QT1 + kTile;  // Q1'(obs'), Q2'(obs'); then the head deltas
  float *QS1 = QT2 + kTile, *QS2 = QS1 + kTile;  // Q1(obs), Q2(obs)
  float *D0 = QS2 + kTile, *D1 = D0 + kTile;   // deltas (the obs' forwards: scratch)
  float *H1 = D1 + kTile;                      // Q1 hidden outputs on obs
  float *H2 = H1 + (P.L[1] - 1) * kTile;       // Q2 hidden outputs on obs

  load_net(Wa, U.actor, P, 0);
  load_net(Wc1, U.critic, P, 1);
  load_net(Wc2, U.critic2, P, 1);
  load_net(Wt1, U.target_critic, P, 1);
  load_net(Wt2, U.target_critic2, P, 1);
  for (int e = tid; e < g_total; e += kThreads) G1[e] = 0.0f;
  for (int e = tid; e < P.n_buf * kTile; e += kThreads) X[e] = 0.0f;
  __syncthreads();

  const int F = U.obs_dim, A = U.n_actions, ns = U.n_step, La = P.L[0], Lq = P.L[1];
  const SampledRows rows = {windows, U.capacity};
  const long long EN = P.EN, M = P.M, E = U.n_envs, Np = U.n_agents;
  const float gamma = U.gamma, alpha = expf(*U.log_alpha);
  const float norm_q = (float)(2.0 / (double)M);        // mse_loss backward: 2 / numel
  double e1_acc = 0.0, e2_acc = 0.0;

  for (long long g0 = (long long)blockIdx.x * kRows; g0 < M; g0 += (long long)gridDim.x * kRows) {
    for (int e = tid; e < kRows * F; e += kThreads) {
      const int r = e / F, c = e - r * F;
      const long long g = g0 + r;
      float x = 0.0f, xb = 0.0f;
      if (g < M) {
        const Row w = rows.at(g);
        x = U.obs[((long long)rows.slot(w, 0) * EN + w.n) * F + c];
        xb = U.obs[((long long)rows.slot(w, ns) * EN + w.n) * F + c];
      }
      X[r * kPitch + c] = x;
      XB[r * kPitch + c] = xb;
    }
    __syncthreads();
    net_forward(Wa, P, 0, XB, [&](int l) { return l == La - 1 ? Z : (l % 2 == 0 ? D0 : D1); });
    net_forward(Wt1, P, 1, XB, [&](int l) { return l == Lq - 1 ? QT1 : (l % 2 == 0 ? D0 : D1); });
    net_forward(Wt2, P, 1, XB, [&](int l) { return l == Lq - 1 ? QT2 : (l % 2 == 0 ? D0 : D1); });
    net_forward(Wc1, P, 1, X, [&](int l) { return l == Lq - 1 ? QS1 : H1 + l * kTile; });
    net_forward(Wc2, P, 1, X, [&](int l) { return l == Lq - 1 ? QS2 : H2 + l * kTile; });
    // ---- per row: V' from the log-softmax, the n-step return, the two head deltas
    if (tid < kRows) {
      const int r = tid;
      const long long g = g0 + r;
      float *d1 = QT1 + r * kPitch, *d2 = QT2 + r * kPitch;
      int a = -1;
      float dq1 = 0.0f, dq2 = 0.0f;
      if (g < M) {
        const Row w = rows.at(g);
        a = U.actions[(long long)rows.slot(w, 0) * EN + w.n];
        const float *z = Z + r * kPitch;
        float mx = z[0];
        for (int c = 1; c < A; c++) mx = fmaxf(mx, z[c]);
        float s = 0.0f;
        for (int c = 0; c < A; c++) s += expf(z[c] - mx);
        const float ls = logf(s);
        float v = 0.0f;
        for (int c = 0; c < A; c++) {
          const float lp = (z[c] - mx) - ls;           // log pi'_c: never log of a softmax
          v = fmaf(expf(lp), fminf(d1[c], d2[c]) - alpha * lp, v);
        }
        const long long env = w.n / Np;
        float ret = v;
        for (int j = ns - 1; j >= 0; j--) {
          const int pk = rows.slot(w, j);
          const float om = U.done[(long long)pk * E + env] != 0 ? 0.0f : 1.0f;
          ret = __fadd_rn(__fmul_rn(__fmul_rn(om, gamma), ret),
                          U.rewards[(long long)pk * EN + w.n]);
        }
        if (U.returns) U.returns[g] = ret;
        // (an action outside [0, A) -- never written by the samplers -- contributes nothing)
        if (a >= 0 && a < A) {
          const float q1 = QS1[r * kPitch + a], q2 = QS2[r * kPitch + a];
          const float e1 = __fsub_rn(q1, ret), e2 = __fsub_rn(q2, ret);
          dq1 = __fmul_rn(e1, norm_q);
          dq2 = __fmul_rn(e2, norm_q);
          e1_acc += (double)e1 * (double)e1;
          e2_acc += (double)e2 * (double)e2;
          if (U.q1_values) U.q1_values[g] = q1;
          if (U.q2_values) U.q2_values[g] = q2;
        } else {
          a = -1;
        }
      }
      for (int c = 0; c < A; c++) {
        d1[c] = 0.0f;
        d2[c] = 0.0f;
      }
      if (a >= 0) {
        d1[a] = dq1;
        d2[a] = dq2;
      }
    }
    __syncthreads();
    net_backward(Wc1, P, 1, G1, QT1, [&](int l) { return l == 0 ? X : H1 + (l - 1) * kTile; },
                 D0, D1, -1);
    net_backward(Wc2, P, 1, G2, QT2, [&](int l) { return l == 0 ? X : H2 + (l - 1) * kTile; },
                 D0, D1, -1);
  }
  write_partials(G1, g_total, e1_acc, e2_acc, s_e1, s_e2, partials, psums);
}

// Actor pass: the gradient of (1/B) sum_g sum_a pi_a (alpha log pi_a - min(Q1, Q2)_a) into
// per-CTA actor partials; psums: sum_g sum_a pi_a min(Q1, Q2)_a, sum_g sum_a pi_a log pi_a.
__global__ void __launch_bounds__(kThreads, 1)
sac_discrete_actor_kernel(const __grid_constant__ wdb_sac_discrete_update_args U,
                          const __grid_constant__ Plan Pg, float *partials, double *psums,
                          const int2 *windows) {
  extern __shared__ __align__(16) float smem[];
  __shared__ Plan P;
  __shared__ double s_q[kRows], s_lp[kRows];
  if (threadIdx.x == 0) P = Pg;
  __syncthreads();
  const int tid = threadIdx.x;
  float *Wa = smem, *Wc1 = Wa + P.wfloats[0], *Wc2 = Wc1 + P.wfloats[1];
  float *Ga = Wc2 + P.wfloats[1];
  const int g_total = P.gfloats[0];
  float *X = Ga + ((g_total + 3) / 4) * 4;     // obs at slot(0)
  float *Z = X + kTile;                        // actor logits; then the logit deltas
  float *QS1 = Z + kTile, *QS2 = QS1 + kTile;  // Q1(obs), Q2(obs)
  float *D0 = QS2 + kTile, *D1 = D0 + kTile;   // deltas (the critic forwards: scratch)
  float *HA = D1 + kTile;                      // actor hidden outputs

  load_net(Wa, U.actor, P, 0);
  load_net(Wc1, U.critic, P, 1);
  load_net(Wc2, U.critic2, P, 1);
  for (int e = tid; e < g_total; e += kThreads) Ga[e] = 0.0f;
  for (int e = tid; e < P.n_buf * kTile; e += kThreads) X[e] = 0.0f;
  __syncthreads();

  const int F = U.obs_dim, A = U.n_actions, La = P.L[0], Lq = P.L[1];
  const SampledRows rows = {windows, U.capacity};
  const long long EN = P.EN, M = P.M;
  const float alpha = expf(*U.log_alpha);
  const float inv_b = (float)(1.0 / (double)M);
  double q_acc = 0.0, lp_acc = 0.0;

  for (long long g0 = (long long)blockIdx.x * kRows; g0 < M; g0 += (long long)gridDim.x * kRows) {
    for (int e = tid; e < kRows * F; e += kThreads) {
      const int r = e / F, c = e - r * F;
      const long long g = g0 + r;
      float x = 0.0f;
      if (g < M) {
        const Row w = rows.at(g);
        x = U.obs[((long long)rows.slot(w, 0) * EN + w.n) * F + c];
      }
      X[r * kPitch + c] = x;
    }
    __syncthreads();
    net_forward(Wa, P, 0, X, [&](int l) { return l == La - 1 ? Z : HA + l * kTile; });
    net_forward(Wc1, P, 1, X, [&](int l) { return l == Lq - 1 ? QS1 : (l % 2 == 0 ? D0 : D1); });
    net_forward(Wc2, P, 1, X, [&](int l) { return l == Lq - 1 ? QS2 : (l % 2 == 0 ? D0 : D1); });
    // ---- per row: the log-softmax, h = alpha log pi - min(Q1, Q2), the logit delta
    if (tid < kRows) {
      const int r = tid;
      const long long g = g0 + r;
      float *z = Z + r * kPitch;
      const float *q1 = QS1 + r * kPitch, *q2 = QS2 + r * kPitch;
      if (g < M) {
        float mx = z[0];
        for (int c = 1; c < A; c++) mx = fmaxf(mx, z[c]);
        float s = 0.0f;
        for (int c = 0; c < A; c++) s += expf(z[c] - mx);
        const float ls = logf(s);
        float hbar = 0.0f, pm = 0.0f, plp = 0.0f;
        for (int c = 0; c < A; c++) {
          const float lp = (z[c] - mx) - ls, pi = expf(lp), m = fminf(q1[c], q2[c]);
          hbar = fmaf(pi, alpha * lp - m, hbar);
          pm = fmaf(pi, m, pm);
          plp = fmaf(pi, lp, plp);
        }
        for (int c = 0; c < A; c++) {
          const float lp = (z[c] - mx) - ls, pi = expf(lp), m = fminf(q1[c], q2[c]);
          z[c] = pi * ((alpha * lp - m) - hbar) * inv_b;
        }
        q_acc += (double)pm;
        lp_acc += (double)plp;
        if (U.entropies) U.entropies[g] = -plp;
      } else {
        for (int c = 0; c < A; c++) z[c] = 0.0f;
      }
    }
    __syncthreads();
    net_backward(Wa, P, 0, Ga, Z, [&](int l) { return l == 0 ? X : HA + (l - 1) * kTile; }, D0,
                 D1, -1);
  }
  write_partials(Ga, g_total, q_acc, lp_acc, s_q, s_lp, partials, psums);
}

// Launches one pass over w's windows and the reduction of its per-CTA partials into the trained
// networks' gradients and u->sums (the critic pass's two, then the actor pass's two).
int sac_discrete_update(void *stream, const wdb_sac_discrete_update_args *u,
                        const wdb_replay_windows *w, bool actor_pass) {
  Plan P;
  if (!sac_discrete_plan(u, w, actor_pass, &P)) return (int)cudaErrorInvalidValue;
  if (!w->windows || !u->obs || !u->log_alpha || !u->workspace) return (int)cudaErrorInvalidValue;
  if (!net_ok(u->actor, P.L[0], actor_pass) || !net_ok(u->critic, P.L[1], !actor_pass) ||
      !net_ok(u->critic2, P.L[1], !actor_pass))
    return (int)cudaErrorInvalidValue;
  if (!actor_pass && (!u->actions || !u->rewards || !u->done ||
                      !net_ok(u->target_critic, P.L[1], false) ||
                      !net_ok(u->target_critic2, P.L[1], false)))
    return (int)cudaErrorInvalidValue;
  Reduce R = {};
  int widest = 1;
  if (actor_pass) {
    R.g_total = P.gfloats[0];
    add_segments(&R, P, 0, 0, u->actor, &widest);
  } else {
    R.g_total = 2 * P.gfloats[1];
    add_segments(&R, P, 1, 0, u->critic, &widest);
    add_segments(&R, P, 1, P.gfloats[1], u->critic2, &widest);
  }
  static size_t configured[2] = {0, 0};
  const void *kernel = actor_pass ? (const void *)sac_discrete_actor_kernel
                                  : (const void *)sac_discrete_critic_kernel;
  const size_t smem = (size_t)P.smem_floats * sizeof(float);
  int rc = allow_smem(kernel, smem, &configured[actor_pass ? 1 : 0]);
  if (rc != cudaSuccess) return rc;
  double *psums = static_cast<double *>(u->workspace);
  float *partials = reinterpret_cast<float *>(psums + 2 * P.grid);
  const int2 *windows = reinterpret_cast<const int2 *>(w->windows);
  if (actor_pass)
    sac_discrete_actor_kernel<<<P.grid, kThreads, smem, as_stream(stream)>>>(*u, P, partials,
                                                                             psums, windows);
  else
    sac_discrete_critic_kernel<<<P.grid, kThreads, smem, as_stream(stream)>>>(*u, P, partials,
                                                                              psums, windows);
  rc = finish_launch();
  if (rc != cudaSuccess) return rc;
  R.grid = P.grid;
  double *sums = u->sums ? u->sums + (actor_pass ? 2 : 0) : nullptr;
  return launch_reduce(stream, R, widest, partials, psums, sums);
}

}  // namespace

// ---------------------------------------------------------------------------- entry points
#define WDB_SAC_DISCRETE_API(pass, actor_pass)                                                  \
  WDB_API int wdb_sac_discrete_##pass##_update_sampled_supported(                               \
      const wdb_sac_discrete_update_args *u, int n_windows) {                                  \
    const wdb_replay_windows w = {nullptr, n_windows};                                         \
    Plan P;                                                                                    \
    return sac_discrete_plan(u, &w, actor_pass, &P) ? 1 : 0;                                   \
  }                                                                                            \
  WDB_API long long wdb_sac_discrete_##pass##_update_sampled_workspace_bytes(                   \
      const wdb_sac_discrete_update_args *u, int n_windows) {                                  \
    const wdb_replay_windows w = {nullptr, n_windows};                                         \
    Plan P;                                                                                    \
    return sac_discrete_plan(u, &w, actor_pass, &P) ? sac_discrete_workspace_bytes(P, actor_pass) \
                                                    : -1;                                      \
  }                                                                                            \
  WDB_API int wdb_sac_discrete_##pass##_update_sampled(                                         \
      void *stream, const wdb_sac_discrete_update_args *u, const wdb_replay_windows *w) {       \
    return w ? sac_discrete_update(stream, u, w, actor_pass) : (int)cudaErrorInvalidValue;     \
  }

WDB_SAC_DISCRETE_API(critic, false)
WDB_SAC_DISCRETE_API(actor, true)
