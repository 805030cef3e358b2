// wdb_dqn_pass.cuh -- DQN's replay-update tile body and its plan (QR-DQN's at N = 1), shared by
// wdb_ddpg_update.cu (dqn_pass_kernel, dqn_weighted_kernel, and QR-DQN's plan),
// wdb_masked_q.cu (the action-masked kernels) and wdb_branching_q.cu (the action-branching
// kernels).  kMasked = kBranching = false is the code the pinned kernels were compiled from; the
// masked bootstrap and the branching bootstrap and gradient sit under `if constexpr`.
#pragma once

#include "wdb_common.cuh"
#include "wdb_update_tiles.cuh"

namespace {

using namespace wdb;

// QR-DQN's plan, and DQN's at N = 1: the online and target Q networks in the actor-shaped slot
// (input F, head A * N <= 64).  plan_layout also lays out a critic-shaped slot, which the Q
// passes do not use: it is given an action width of 1, so its input F + 1 only asks F <= 63 of
// the Q network (F + A is no limit).  The kernel holds both networks, their gradient block and
// 8 + (hidden layers) row tiles.
bool qr_dqn_plan(const wdb_dqn_update_args *u, int nq, const wdb_replay_windows *w, Plan *p) {
  if (!u || !w || !(u->huber_delta > 0.0f)) return false;
  if (nq < 1 || nq > kMaxWidth || u->n_actions < 1 || u->n_actions > kMaxWidth) return false;
  const wdb_ddpg_net *qs[2] = {&u->q, &u->target_q};
  const wdb_ddpg_net *const *nets[2] = {qs, qs};
  const int count[2] = {2, 2};
  if (!plan_layout(u->n_envs, u->n_agents, u->obs_dim, 1, u->n_actions * nq, u->capacity, 0,
                   u->n_step, w, nets, count, p))
    return false;
  return plan_smem(p, 8 + (p->L[0] - 1), 2ll * p->wfloats[0], p->gfloats[0]);
}

long long dqn_workspace_bytes(const Plan &P) { return 16ll * P.grid + 4ll * P.grid * P.gfloats[0]; }

// wdb_dqn_update_sampled's tile kernel: the online and target Q networks in the actor-shaped
// Plan slot (head = A).  Per tile of kRows sampled windows: online Q(obs) (its hidden outputs
// kept for the backward), target Q'(obs') and, with double_q, online Q(obs'); per row the
// bootstrap, the n-step return and the Huber gradient in the action's column; then back
// through the online network.  Kernels of their own, so the DDPG, TD3 and SAC kernels keep their
// code.
// kWeighted (wdb_dqn_update_prioritized): row g's Huber value and clamped difference are scaled
// by weights[g] -- the clamped difference before the 1 / B, so a weight of 1 changes no bit.
// kMasked (wdb_dqn_update_masked): the bootstrap's a* (double_q) or max ranges over the valid
// actions of action_mask [C, E, Np, A] at the window's slot(n_step), read by the row's own
// thread; a row with no valid action takes every action.  The first maximum among the valid
// actions is the first maximum overall when every action is valid, so an all-ones mask gives
// the unmasked pass's bits.
// kBranching (wdb_branching_dqn_update_sampled / _prioritized): the head holds D branches
// (*branches), the row's D actions sit at actions[(slot(0) * EN + n) * D + d], the bootstrap is
// the mean over the branches of each branch's DQN bootstrap, and each valid branch action gets
// the Huber gradient against the shared return, scaled by 1 / (B D); the loss row and Q-bar are
// the means over the branches.  Every divide by D is exact at D = 1: DQN's bits.
template <bool kWeighted, bool kMasked = false, bool kBranching = false>
__device__ __forceinline__ void dqn_tile_pass(const wdb_dqn_update_args &U, const Plan &Pg,
                                              float *partials, double *psums,
                                              const int2 *windows, const float *weights,
                                              const float *action_mask = nullptr,
                                              const wdb_q_branches *branches = nullptr) {
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
  float *XB = X + kTile;                       // bootstrap obs at slot(n_step)
  float *QS = XB + kTile;                      // online Q(obs)
  float *QT = QS + kTile;                      // target Q'(obs')
  float *QD = QT + kTile;                      // online Q(obs') (double_q)
  float *DQ = QD + kTile;                      // head delta
  float *D0 = DQ + kTile, *D1 = D0 + kTile;    // deltas (the obs' forwards: scratch)
  float *H = D1 + kTile;                       // online hidden outputs on obs

  load_net(Wq, U.q, P, 0);
  load_net(Wt, U.target_q, P, 0);
  for (int e = tid; e < g_total; e += kThreads) G[e] = 0.0f;
  for (int e = tid; e < P.n_buf * kTile; e += kThreads) X[e] = 0.0f;
  __syncthreads();

  const int F = U.obs_dim, A = U.n_actions, L = P.L[0], ns = U.n_step;
  const SampledRows rows = {windows, U.capacity};
  const long long EN = P.EN, M = P.M, E = U.n_envs, Np = U.n_agents;
  const float gamma = U.gamma, delta = U.huber_delta;
  const float norm = (float)(1.0 / (double)M);           // huber_loss backward, mean: 1 / numel
  double h_acc = 0.0, q_acc = 0.0;

  for (long long g0 = (long long)blockIdx.x * kRows; g0 < M; g0 += (long long)gridDim.x * kRows) {
    // ---- inputs: X = obs at slot(0), XB = obs at slot(n_step)
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
    net_forward(Wq, P, 0, X, [&](int l) { return l == L - 1 ? QS : H + l * kTile; });
    net_forward(Wt, P, 0, XB, [&](int l) { return l == L - 1 ? QT : (l % 2 == 0 ? D0 : D1); });
    if (U.double_q)
      net_forward(Wq, P, 0, XB, [&](int l) { return l == L - 1 ? QD : (l % 2 == 0 ? D0 : D1); });
    // ---- bootstrap, n-step return (done != 0 is terminal) and the Huber gradient
    if (tid < kRows) {
      const int r = tid;
      const long long g = g0 + r;
      float *dq = DQ + r * kPitch;
      for (int c = 0; c < A; c++) dq[c] = 0.0f;
      if (g < M) {
        const Row w = rows.at(g);
        const int a = kBranching ? 0 : U.actions[(long long)rows.slot(w, 0) * EN + w.n];
        const float *qt = QT + r * kPitch;
        float boot;
        if constexpr (kBranching) {
          // per branch: the target's value of the online first argmax, or the target's max
          // (its value at the target's own first argmax); then their mean
          const float *qc = U.double_q ? QD + r * kPitch : qt;
          const int D = branches->n_heads;
          float sum = 0.0f;
          for (int d = 0, o = 0; d < D; o += branches->sizes[d], d++) {
            float best = qc[o];
            int k = o;
            for (int c = o + 1; c < o + branches->sizes[d]; c++)
              if (best < qc[c]) { best = qc[c]; k = c; }
            sum = d == 0 ? qt[k] : __fadd_rn(sum, qt[k]);
          }
          boot = __fdiv_rn(sum, (float)D);
        } else if constexpr (kMasked) {
          // a* over the valid actions of obs' own mask (slot n_step); none valid: every action
          const float *mk = action_mask + ((long long)rows.slot(w, ns) * EN + w.n) * A;
          bool any = false;
          for (int c = 0; c < A; c++) any |= mk[c] != 0.0f;
          const float *qc = U.double_q ? QD + r * kPitch : qt;
          float best = 0.0f;
          int k = -1;
          for (int c = 0; c < A; c++)
            if ((!any || mk[c] != 0.0f) && (k < 0 || best < qc[c])) { best = qc[c]; k = c; }
          boot = qt[k];
        } else if (U.double_q) {               // the target's value of the online first argmax
          const float *qd = QD + r * kPitch;
          float best = qd[0];
          int k = 0;
          for (int c = 1; c < A; c++)
            if (best < qd[c]) { best = qd[c]; k = c; }
          boot = qt[k];
        } else {
          boot = qt[0];
          for (int c = 1; c < A; c++)
            if (boot < qt[c]) boot = qt[c];
        }
        const long long env = w.n / Np;
        float ret = boot;
        for (int j = ns - 1; j >= 0; j--) {
          const int pk = rows.slot(w, j);
          const float om = U.done[(long long)pk * E + env] != 0 ? 0.0f : 1.0f;
          ret = __fadd_rn(__fmul_rn(__fmul_rn(om, gamma), ret),
                          U.rewards[(long long)pk * EN + w.n]);
        }
        if constexpr (kBranching) {
          // (a branch action outside [0, A_d) -- never written by the samplers -- contributes
          // nothing)
          const int D = branches->n_heads;
          const float nd = (float)(1.0 / ((double)M * (double)D));
          const int *acts = U.actions + ((long long)rows.slot(w, 0) * EN + w.n) * D;
          double h_row = 0.0;
          float q_sum = 0.0f;
          bool any = false;
          for (int d = 0, o = 0; d < D; o += branches->sizes[d], d++) {
            const int ab = acts[d];
            if (ab < 0 || ab >= branches->sizes[d]) continue;
            const float q = QS[r * kPitch + o + ab];
            const float diff = __fsub_rn(q, ret);
            const double ad = fabs((double)diff);
            if constexpr (kWeighted) {
              const float w = weights[g];
              const double wd = (double)w;
              dq[o + ab] = __fmul_rn(__fmul_rn(fminf(fmaxf(diff, -delta), delta), w), nd);
              h_row += ad < (double)delta ? (0.5 * wd) * ad * ad
                                          : (wd * (double)delta) * (ad - 0.5 * (double)delta);
            } else {
              dq[o + ab] = __fmul_rn(fminf(fmaxf(diff, -delta), delta), nd);
              h_row += ad < (double)delta ? 0.5 * ad * ad
                                          : (double)delta * (ad - 0.5 * (double)delta);
            }
            q_sum = any ? __fadd_rn(q_sum, q) : q;
            any = true;
          }
          if (any) {
            const float q_bar = __fdiv_rn(q_sum, (float)D);
            h_acc += h_row / (double)D;
            q_acc += (double)q_bar;
            if (U.q_values) U.q_values[g] = q_bar;
          }
        } else if (a >= 0 && a < A) {
          // (an action outside [0, A) -- never written by the samplers -- contributes nothing)
          const float q = QS[r * kPitch + a];
          const float diff = __fsub_rn(q, ret);
          const double ad = fabs((double)diff);
          if constexpr (kWeighted) {
            const float w = weights[g];
            const double wd = (double)w;
            dq[a] = __fmul_rn(__fmul_rn(fminf(fmaxf(diff, -delta), delta), w), norm);
            h_acc += ad < (double)delta ? (0.5 * wd) * ad * ad
                                        : (wd * (double)delta) * (ad - 0.5 * (double)delta);
          } else {
            dq[a] = __fmul_rn(fminf(fmaxf(diff, -delta), delta), norm);
            h_acc += ad < (double)delta ? 0.5 * ad * ad
                                        : (double)delta * (ad - 0.5 * (double)delta);
          }
          q_acc += (double)q;
          if (U.q_values) U.q_values[g] = q;
        }
        if (U.returns) U.returns[g] = ret;
      }
    }
    __syncthreads();
    net_backward(Wq, P, 0, G, DQ, [&](int l) { return l == 0 ? X : H + (l - 1) * kTile; }, D0,
                 D1, -1);
  }

  // ---- this CTA's partials
  float *part = partials + (long long)blockIdx.x * g_total;
  for (int e = tid; e < g_total; e += kThreads) part[e] = G[e];
  if (tid < kRows) {
    s_h[tid] = h_acc;
    s_q[tid] = q_acc;
  }
  __syncthreads();
  if (tid == 0) {
    double a = 0.0, b = 0.0;
    for (int r = 0; r < kRows; r++) {
      a += s_h[r];
      b += s_q[r];
    }
    psums[2 * blockIdx.x] = a;
    psums[2 * blockIdx.x + 1] = b;
  }
}

}  // namespace
