// wdb_tqc.cu -- one TQC update (Kuznetsov et al. 2020, "Controlling Overestimation Bias with
// Truncated Mixture of Continuous Distributional Quantile Critics") of one policy over B sampled
// replay windows, as two passes of two launches each: a tile kernel and the fixed-order
// reduction of its per-CTA partials (include/wdb200.h, wdb_tqc_{critic,actor}_update_sampled).
//
// The actor is SAC's squashed Gaussian (squashed_dim); the two critics and their targets map
// obs ++ action to N quantiles.  In a row tile, critic m's N columns start at column m * NC, NC =
// N rounded up to a multiple of 4, so each critic's head delta is float4-aligned for its own
// backward.
//   critic pass, per tile of kRows windows: the actor on obs' -> a' and the log-prob terms; both
//     target critics on (obs', a') into one tile of 2N atoms; per row, on its 16 threads (thread
//     k owns the pooled atoms j = k mod 16), each atom's rank among the row's 2N by comparison
//     (ties to the lower pooled index: a stable sort), and the n-step return of each kept atom
//     (rank < K) written at its rank into a second tile; both critics on (obs, a) into a third
//     tile (hidden outputs kept); per row the quantile Huber pair loss, thread k owning the
//     (m, i) = k mod 16 and summing over the K returns in ascending order, d theta written in
//     place; then back through each critic into its own gradient block.
//   actor pass, per tile: the actor (hidden outputs kept) -> a; both critics on (obs, a); per
//     row d theta = -1 / (B 2 N) in every quantile column, back through each critic to its action
//     inputs (no critic weight gradient); then SAC's tail: the tanh, the reparameterisation, the
//     log-prob's own terms and the clamp, back through the actor.
// The per-row sums over a row's 16 threads are xor butterflies (the same bits in every lane), the
// partials are reduced in CTA order, and there are no float atomics: a relaunch is bit-identical.
// Its own translation unit, on the primitives of wdb_update_tiles.cuh, so every other update
// kernel keeps its machine code.
#include "wdb_common.cuh"
#include "wdb_update_tiles.cuh"
#include "wdb_sac_terms.cuh"             // sampled_return, squashed_dim

using namespace wdb;

namespace {

constexpr int kCritics = 2;                   // the native passes' M
constexpr int kLanes = kThreads / kRows;      // threads per loss row

// The first column of critic 1's quantiles in a tile (critic 0's start at column 0).
__host__ __device__ __forceinline__ int head_col(int N) { return (N + 3) & ~3; }

// The plan of one pass: SAC's (the actor shape with head 2A, the critic shape for the four
// critics), then the critic head set to N.  The critic pass holds the actor, four critics, both
// critic gradient blocks and 8 + 2 (hidden layers) row tiles; the actor pass the actor, both
// critics, the actor gradient block and 6 + 2 (critic hidden layers) + (actor hidden layers).
bool tqc_plan(const wdb_tqc_update_args *u, const wdb_replay_windows *w, bool actor_pass,
              Plan *p) {
  if (!u || !w) return false;
  if (!(u->log_std_min <= u->log_std_max)) return false;
  const int N = u->n_quantiles;
  if (N < 2 || 2 * N > kMaxWidth || u->n_drop < 0 || u->n_drop >= N) return false;
  const wdb_ddpg_net *actors[1] = {&u->actor};
  const wdb_ddpg_net *critics[4] = {&u->critic, &u->critic2, &u->target_critic,
                                    &u->target_critic2};
  const wdb_ddpg_net *const *nets[2] = {actors, critics};
  const int count[2] = {1, 4};
  if (!plan_layout(u->n_envs, u->n_agents, u->obs_dim, u->action_dim, 2 * u->action_dim,
                   u->capacity, 0, u->n_step, w, nets, count, p))
    return false;
  const int L = p->L[1], hin = p->in[1][L - 1], pw = p->pw[1][L - 1];
  p->out[1][L - 1] = N;
  p->wfloats[1] = p->woff[1][L - 1] + round_up(N * pw + N, 4);
  p->gfloats[1] = p->goff[1][L - 1] + N * hin + N;
  if (actor_pass)
    return plan_smem(p, 6 + 2 * (L - 1) + (p->L[0] - 1), p->wfloats[0] + 2ll * p->wfloats[1],
                     p->gfloats[0]);
  return plan_smem(p, 8 + 2 * (L - 1), p->wfloats[0] + 4ll * p->wfloats[1], 2 * p->gfloats[1]);
}

long long tqc_workspace_bytes(const Plan &P, bool actor_pass) {
  return 16ll * P.grid + 4ll * P.grid * (actor_pass ? P.gfloats[0] : 2 * P.gfloats[1]);
}

// The sum of x over the kLanes threads of a loss row, the same bits in each of them.
__device__ __forceinline__ double row_sum(double x) {
#pragma unroll
  for (int off = kLanes / 2; off > 0; off /= 2) x += __shfl_xor_sync(0xffffffffu, x, off);
  return x;
}

// Writes this CTA's gradient block and the sums of a_acc and b_acc over the kRows threads that
// accumulate them (slot: 0 .. kRows - 1 for those, -1 for the others), in slot order.
__device__ __forceinline__ void write_partials(const float *G, int g_total, double a_acc,
                                               double b_acc, int slot, float *partials,
                                               double *psums) {
  __shared__ double s_a[kRows], s_b[kRows];
  const int tid = threadIdx.x;
  float *part = partials + (long long)blockIdx.x * g_total;
  for (int e = tid; e < g_total; e += kThreads) part[e] = G[e];
  if (slot >= 0) {
    s_a[slot] = a_acc;
    s_b[slot] = b_acc;
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

// Critic pass: the gradients of the truncated quantile Huber loss into per-CTA partials
// [G1 | G2]; psums: sum_g loss_g, sum_g mean theta.
__global__ void __launch_bounds__(kThreads, 1)
tqc_critic_kernel(const __grid_constant__ wdb_tqc_update_args U, const __grid_constant__ Plan Pg,
                  float *partials, double *psums, const int2 *windows) {
  extern __shared__ __align__(16) float smem[];
  __shared__ Plan P;
  if (threadIdx.x == 0) P = Pg;
  __syncthreads();
  const int tid = threadIdx.x;
  float *Wa = smem, *Wc1 = Wa + P.wfloats[0], *Wc2 = Wc1 + P.wfloats[1];
  float *Wt1 = Wc2 + P.wfloats[1], *Wt2 = Wt1 + P.wfloats[1];
  float *G1 = Wt2 + P.wfloats[1], *G2 = G1 + P.gfloats[1];
  const int g_total = 2 * P.gfloats[1];
  float *XQ = G1 + ((g_total + 3) / 4) * 4;    // obs ++ actions at slot(0)
  float *XB = XQ + kTile;                      // obs' ++ a' at slot(n_step)
  float *Z = XB + kTile;                       // actor head on obs'; then [0, A): log-prob terms
  float *D0 = Z + kTile, *D1 = D0 + kTile;     // deltas (the obs' forwards: scratch)
  float *ZT = D1 + kTile;                      // the pooled target atoms
  float *Y = ZT + kTile;                       // the kept atoms' returns T_0 .. T_{K-1}
  float *TH = Y + kTile;                       // theta of both critics on (obs, a); then d theta
  float *H1 = TH + kTile;                      // critic hidden outputs on (obs, a)
  float *H2 = H1 + (P.L[1] - 1) * kTile;       // critic2 hidden outputs on (obs, a)

  load_net(Wa, U.actor, P, 0);
  load_net(Wc1, U.critic, P, 1);
  load_net(Wc2, U.critic2, P, 1);
  load_net(Wt1, U.target_critic, P, 1);
  load_net(Wt2, U.target_critic2, P, 1);
  for (int e = tid; e < g_total; e += kThreads) G1[e] = 0.0f;
  for (int e = tid; e < P.n_buf * kTile; e += kThreads) XQ[e] = 0.0f;
  __syncthreads();

  const int F = U.obs_dim, A = U.action_dim, FA = F + A, ns = U.n_step;
  const int La = P.L[0], Lq = P.L[1];
  const int N = U.n_quantiles, NC = head_col(N), K = kCritics * (N - U.n_drop);
  const SampledRows rows = {windows, U.capacity};
  const long long EN = P.EN, B = P.M;
  const float scale = U.action_scale, bias = U.action_bias;
  const float lo = U.log_std_min, hi = U.log_std_max;
  const float alpha = expf(*U.log_alpha);
  const float c_loss = (float)(1.0 / ((double)B * kCritics * N * K));
  const int r = tid / kLanes, k = tid % kLanes;   // this thread's row of the tile and lane
  double l_acc = 0.0, q_acc = 0.0;

  for (long long g0 = (long long)blockIdx.x * kRows; g0 < B; g0 += (long long)gridDim.x * kRows) {
    // ---- inputs: XQ = obs ++ actions at slot(0), XB = obs at slot(n_step)
    for (int e = tid; e < kRows * FA; e += kThreads) {
      const int rr = e / FA, c = e - rr * FA;
      const long long g = g0 + rr;
      float xq = 0.0f, xb = 0.0f;
      if (g < B) {
        const Row w = rows.at(g);
        const long long row = (long long)rows.slot(w, 0) * EN + w.n;
        if (c < F) {
          xq = U.obs[row * F + c];
          xb = U.obs[((long long)rows.slot(w, ns) * EN + w.n) * F + c];
        } else {
          xq = U.actions[row * A + (c - F)];
        }
      }
      XQ[rr * kPitch + c] = xq;
      if (c < F) XB[rr * kPitch + c] = xb;
    }
    __syncthreads();
    // ---- 1. actor on obs' -> a' ~ pi(. | obs') into XB's action columns, log-prob terms into Z
    net_forward(Wa, P, 0, XB, [&](int l) { return l == La - 1 ? Z : (l % 2 == 0 ? D0 : D1); });
    for (int e = tid; e < kRows * A; e += kThreads) {
      const int rr = e / A, c = e - rr * A;
      const long long g = g0 + rr;
      const float eps = g < B ? U.critic_noise[g * A + c] : 0.0f;
      const SquashedDim s = squashed_dim(Z + rr * kPitch, A, c, eps, lo, hi);
      XB[rr * kPitch + F + c] = __fadd_rn(__fmul_rn(scale, s.y), bias);
      Z[rr * kPitch + c] = s.term;
    }
    __syncthreads();
    // ---- 2. both target critics -> the pooled atoms; 5. both critics on (obs, a) -> theta
    net_forward(Wt1, P, 1, XB, [&](int l) { return l == Lq - 1 ? ZT : (l % 2 == 0 ? D0 : D1); });
    net_forward(Wt2, P, 1, XB,
                [&](int l) { return l == Lq - 1 ? ZT + NC : (l % 2 == 0 ? D0 : D1); });
    net_forward(Wc1, P, 1, XQ, [&](int l) { return l == Lq - 1 ? TH : H1 + l * kTile; });
    net_forward(Wc2, P, 1, XQ, [&](int l) { return l == Lq - 1 ? TH + NC : H2 + l * kTile; });
    // ---- 3., 4. each atom's rank; the kept atoms' returns at their rank
    const long long g = g0 + r;
    const float *zt = ZT + r * kPitch;
    float *y = Y + r * kPitch;
    if (g < B) {
      const Row w = rows.at(g);
      float lp = 0.0f;
      for (int c = 0; c < A; c++) lp += Z[r * kPitch + c];
      const float alp = __fmul_rn(alpha, lp);
      for (int j = k; j < kCritics * N; j += kLanes) {
        const int mj = j / N;
        const float v = zt[mj * NC + (j - mj * N)];
        int rank = 0;
        for (int m = 0; m < kCritics; m++)
          for (int i = 0; i < N; i++) {
            const float x = zt[m * NC + i];
            rank += (x < v || (x == v && m * N + i < j)) ? 1 : 0;
          }
        if (rank < K) y[rank] = sampled_return(U, P, rows, w, __fsub_rn(v, alp));
      }
    }
    __syncthreads();
    // ---- 6. the pair loss and d theta, in place
    double row_l = 0.0, row_q = 0.0, row_t = 0.0;
    float *th = TH + r * kPitch;
    for (int j = k; j < kCritics * N; j += kLanes) {
      const int m = j / N, i = j - m * N, col = m * NC + i;
      float d = 0.0f;
      if (g < B) {
        const float theta = th[col];
        const float tau = __fdiv_rn((float)(2 * i + 1), (float)(2 * N));
        float lsum = 0.0f, gsum = 0.0f;
        for (int kk = 0; kk < K; kk++) {
          const float u = __fsub_rn(y[kk], theta);
          const float au = fabsf(u);
          const float wgt = fabsf(tau - (u < 0.0f ? 1.0f : 0.0f));
          const float h = au <= 1.0f ? 0.5f * u * u : au - 0.5f;
          lsum = fmaf(wgt, h, lsum);
          gsum = fmaf(wgt, fminf(fmaxf(u, -1.0f), 1.0f), gsum);
        }
        d = __fmul_rn(-c_loss, gsum);
        row_l += (double)lsum;
        row_q += (double)theta;
      }
      th[col] = d;
    }
    if (g < B)
      for (int kk = k; kk < K; kk += kLanes) row_t += (double)y[kk];
    row_l = row_sum(row_l);
    row_q = row_sum(row_q);
    row_t = row_sum(row_t);
    if (g < B && k == 0) {
      const double q_mean = row_q / (double)(kCritics * N);
      l_acc += row_l;
      q_acc += q_mean;
      if (U.q_means) U.q_means[g] = (float)q_mean;
      if (U.target_means) U.target_means[g] = (float)(row_t / (double)K);
    }
    __syncthreads();
    // ---- 7. backward: each critic on (obs, a) into its own gradient block
    net_backward(Wc1, P, 1, G1, TH, [&](int l) { return l == 0 ? XQ : H1 + (l - 1) * kTile; },
                 D0, D1, -1);
    net_backward(Wc2, P, 1, G2, TH + NC,
                 [&](int l) { return l == 0 ? XQ : H2 + (l - 1) * kTile; }, D0, D1, -1);
  }
  write_partials(G1, g_total, l_acc, q_acc, k == 0 ? r : -1, partials, psums);
}

// Actor pass: the gradient of (1/B) sum_g (alpha log pi(a | obs) - Qbar_g(obs, a)) into per-CTA
// actor partials; psums: sum_g Qbar_g, sum_g log pi.
__global__ void __launch_bounds__(kThreads, 1)
tqc_actor_kernel(const __grid_constant__ wdb_tqc_update_args U, const __grid_constant__ Plan Pg,
                 float *partials, double *psums, const int2 *windows) {
  extern __shared__ __align__(16) float smem[];
  __shared__ Plan P;
  if (threadIdx.x == 0) P = Pg;
  __syncthreads();
  const int tid = threadIdx.x;
  float *Wa = smem, *Wc1 = Wa + P.wfloats[0], *Wc2 = Wc1 + P.wfloats[1];
  float *Ga = Wc2 + P.wfloats[1];
  const int g_total = P.gfloats[0];
  float *XJ = Ga + ((g_total + 3) / 4) * 4;    // obs ++ a
  float *TH = XJ + kTile;                      // theta of both critics; then d theta
  float *Z = TH + kTile;                       // actor head: mu ++ raw log-std
  float *D0 = Z + kTile, *D1 = D0 + kTile;     // deltas
  float *DA = D1 + kTile;                      // log-prob terms, then critic's action gradient
  float *H1 = DA + kTile;                      // critic hidden outputs on (obs, a)
  float *H2 = H1 + (P.L[1] - 1) * kTile;       // critic2 hidden outputs on (obs, a)
  float *HA = H2 + (P.L[1] - 1) * kTile;       // actor hidden outputs

  load_net(Wa, U.actor, P, 0);
  load_net(Wc1, U.critic, P, 1);
  load_net(Wc2, U.critic2, P, 1);
  for (int e = tid; e < g_total; e += kThreads) Ga[e] = 0.0f;
  for (int e = tid; e < P.n_buf * kTile; e += kThreads) XJ[e] = 0.0f;
  __syncthreads();

  const int F = U.obs_dim, A = U.action_dim, La = P.L[0], Lq = P.L[1];
  const int N = U.n_quantiles, NC = head_col(N);
  const SampledRows rows = {windows, U.capacity};
  const long long EN = P.EN, B = P.M;
  const float scale = U.action_scale, bias = U.action_bias;
  const float lo = U.log_std_min, hi = U.log_std_max;
  const float alpha = expf(*U.log_alpha);
  const float d_q = (float)(-1.0 / ((double)B * kCritics * N));   // d loss / d theta_m,i
  const float d_lp = alpha / (float)B;                             // d loss / d log pi
  double q_acc = 0.0, lp_acc = 0.0;

  for (long long g0 = (long long)blockIdx.x * kRows; g0 < B; g0 += (long long)gridDim.x * kRows) {
    for (int e = tid; e < kRows * F; e += kThreads) {
      const int r = e / F, c = e - r * F;
      const long long g = g0 + r;
      float x = 0.0f;
      if (g < B) {
        const Row w = rows.at(g);
        x = U.obs[((long long)rows.slot(w, 0) * EN + w.n) * F + c];
      }
      XJ[r * kPitch + c] = x;
    }
    __syncthreads();
    // ---- 1. actor -> a into XJ's action columns (log-prob terms into DA); 2. both critics
    net_forward(Wa, P, 0, XJ, [&](int l) { return l == La - 1 ? Z : HA + l * kTile; });
    for (int e = tid; e < kRows * A; e += kThreads) {
      const int r = e / A, c = e - r * A;
      const long long g = g0 + r;
      const float eps = g < B ? U.actor_noise[g * A + c] : 0.0f;
      const SquashedDim s = squashed_dim(Z + r * kPitch, A, c, eps, lo, hi);
      XJ[r * kPitch + F + c] = __fadd_rn(__fmul_rn(scale, s.y), bias);
      DA[r * kPitch + c] = s.term;
    }
    __syncthreads();
    net_forward(Wc1, P, 1, XJ, [&](int l) { return l == Lq - 1 ? TH : H1 + l * kTile; });
    net_forward(Wc2, P, 1, XJ, [&](int l) { return l == Lq - 1 ? TH + NC : H2 + l * kTile; });
    // ---- 3. per row: Qbar, log pi and d theta in every quantile column
    if (tid < kRows) {
      const int r = tid;
      const long long g = g0 + r;
      float *th = TH + r * kPitch;
      float d = 0.0f;
      if (g < B) {
        double q = 0.0;
        for (int m = 0; m < kCritics; m++)
          for (int i = 0; i < N; i++) q += (double)th[m * NC + i];
        float lp = 0.0f;
        for (int c = 0; c < A; c++) lp += DA[r * kPitch + c];
        q_acc += q / (double)(kCritics * N);
        lp_acc += (double)lp;
        if (U.log_probs) U.log_probs[g] = lp;
        d = d_q;
      }
      for (int m = 0; m < kCritics; m++)
        for (int i = 0; i < N; i++) th[m * NC + i] = d;
    }
    __syncthreads();
    // ---- both critics back to their action inputs (critic's kept in DA), summed
    const float *da1 = net_backward<false>(
        Wc1, P, 1, nullptr, TH, [&](int l) { return l == 0 ? XJ : H1 + (l - 1) * kTile; }, D0,
        D1, F);
    for (int e = tid; e < kRows * A; e += kThreads) {
      const int r = e / A, c = e - r * A;
      DA[r * kPitch + c] = da1[r * kPitch + F + c];
    }
    __syncthreads();
    const float *da2 = net_backward<false>(
        Wc2, P, 1, nullptr, TH + NC, [&](int l) { return l == 0 ? XJ : H2 + (l - 1) * kTile; },
        D0, D1, F);
    // ---- 4. the tanh, the reparameterisation, the log-prob's own terms and the clamp
    float *dz = da2 == D0 ? D1 : D0;
    for (int e = tid; e < kRows * A; e += kThreads) {
      const int r = e / A, c = e - r * A;
      const long long g = g0 + r;
      float dmu = 0.0f, dls = 0.0f;
      if (g < B) {
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
  write_partials(Ga, g_total, q_acc, lp_acc, tid < kRows ? tid : -1, partials, psums);
}

// Launches one pass over w's windows and the reduction of its per-CTA partials into the trained
// networks' gradients and u->sums (the critic pass's two, then the actor pass's two).
int tqc_update(void *stream, const wdb_tqc_update_args *u, const wdb_replay_windows *w,
               bool actor_pass) {
  Plan P;
  if (!tqc_plan(u, w, actor_pass, &P)) return (int)cudaErrorInvalidValue;
  if (!w->windows || !u->obs || !u->log_alpha || !u->workspace) return (int)cudaErrorInvalidValue;
  if (!net_ok(u->actor, P.L[0], actor_pass) || !net_ok(u->critic, P.L[1], !actor_pass) ||
      !net_ok(u->critic2, P.L[1], !actor_pass))
    return (int)cudaErrorInvalidValue;
  if (actor_pass ? !u->actor_noise
                 : (!u->actions || !u->rewards || !u->done || !u->critic_noise ||
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
  const void *kernel = actor_pass ? (const void *)tqc_actor_kernel : (const void *)tqc_critic_kernel;
  const size_t smem = (size_t)P.smem_floats * sizeof(float);
  int rc = allow_smem(kernel, smem, &configured[actor_pass ? 1 : 0]);
  if (rc != cudaSuccess) return rc;
  double *psums = static_cast<double *>(u->workspace);
  float *partials = reinterpret_cast<float *>(psums + 2 * P.grid);
  const int2 *windows = reinterpret_cast<const int2 *>(w->windows);
  if (actor_pass)
    tqc_actor_kernel<<<P.grid, kThreads, smem, as_stream(stream)>>>(*u, P, partials, psums,
                                                                    windows);
  else
    tqc_critic_kernel<<<P.grid, kThreads, smem, as_stream(stream)>>>(*u, P, partials, psums,
                                                                     windows);
  rc = finish_launch();
  if (rc != cudaSuccess) return rc;
  R.grid = P.grid;
  double *sums = u->sums ? u->sums + (actor_pass ? 2 : 0) : nullptr;
  return launch_reduce(stream, R, widest, partials, psums, sums);
}

}  // namespace

// ---------------------------------------------------------------------------- entry points
#define WDB_TQC_API(pass, actor_pass)                                                          \
  WDB_API int wdb_tqc_##pass##_update_sampled_supported(const wdb_tqc_update_args *u,          \
                                                        int n_windows) {                       \
    const wdb_replay_windows w = {nullptr, n_windows};                                         \
    Plan P;                                                                                    \
    return tqc_plan(u, &w, actor_pass, &P) ? 1 : 0;                                            \
  }                                                                                            \
  WDB_API long long wdb_tqc_##pass##_update_sampled_workspace_bytes(                           \
      const wdb_tqc_update_args *u, int n_windows) {                                           \
    const wdb_replay_windows w = {nullptr, n_windows};                                         \
    Plan P;                                                                                    \
    return tqc_plan(u, &w, actor_pass, &P) ? tqc_workspace_bytes(P, actor_pass) : -1;          \
  }                                                                                            \
  WDB_API int wdb_tqc_##pass##_update_sampled(void *stream, const wdb_tqc_update_args *u,      \
                                              const wdb_replay_windows *w) {                   \
    return w ? tqc_update(stream, u, w, actor_pass) : (int)cudaErrorInvalidValue;              \
  }

WDB_TQC_API(critic, false)
WDB_TQC_API(actor, true)
