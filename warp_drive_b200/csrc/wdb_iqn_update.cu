// wdb_iqn_update.cu -- one implicit quantile network update (Dabney, Ostrovski, Silver & Munos
// 2018) of one policy over B sampled replay windows, in two launches: a tile kernel and the
// fixed-order reduction of its per-CTA partials (include/wdb200.h, wdb_iqn_update_sampled).
//
// The networks: a trunk psi (the Q network's hidden Linear + ReLU layers, width H), the tau
// embedding phi(tau) = ReLU(E cos(pi c tau) + e), c = 0 .. n_cos - 1, and the raw head Linear(H,
// A) on psi(x) * phi(tau).  Per tile of kRows sampled windows, in shared memory:
//   - the trunks once per row: online on obs (its hidden outputs kept for the backward), target
//     on obs' and, with double_q, online on obs';
//   - a* from the collapsed head: the head on psi(obs') * c-bar, c-bar = mean_k phi(tau~_k) over
//     the K midpoint levels, computed by every CTA at its start for both networks;
//   - the target pairs (row, tau'_j): the target embedding, the merge and the target head give
//     target(obs')[a*] at tau'_j, then DQN's n-step recursion gives T_j;
//   - the online pairs (row, tau_i): theta_i = online(obs)[a] at tau_i;
//   - the row's N x N' quantile Huber pairs, spread over the row's 16 threads as QR-DQN's pass
//     spreads them (thread k owns i = k, k + 16, ... and sums over j in order);
//   - the backward over the online pairs again, the embedding recomputed rather than stored:
//     head gradient summed over the pairs, d psi summed over the row's tau's in order, d phi
//     through the ReLU and the cosine features into the embedding's gradient; then d psi back
//     through the trunk.
// Every sum runs in a fixed order and the partials are reduced in CTA order: an update is
// bit-reproducible.  Its own translation unit, on the primitives of wdb_update_tiles.cuh, so the
// kernels of wdb_ddpg_update.cu keep their machine code.
#include "wdb_common.cuh"
#include "wdb_update_tiles.cuh"

using namespace wdb;

namespace {

constexpr int kMaxQuantileSamples = 256;   // K

// The cosine features of one tile of levels: CF[r][c] = cos(freq[c] * tau(r)) for c < n_cos,
// freq[c] = float(pi * c) -- the float32 operations of FullyConnectedIQN.cos_features.
template <class Tau>
__device__ __forceinline__ void cos_features(float *CF, const float *freq, int n_cos, Tau tau) {
  for (int e = threadIdx.x; e < kRows * n_cos; e += kThreads) {
    const int r = e / n_cos, c = e - r * n_cos;
    CF[r * kPitch + c] = cosf(__fmul_rn(tau(r), freq[c]));
  }
}

// The tau embedding of one tile: PHI = ReLU(E CF + e) (net slot 1 of the Plan).
__device__ __forceinline__ void embed(const float *We, const Plan &P, const float *CF, float *PHI) {
  layer_forward(We, P.pw[1][0], P.in[1][0], P.out[1][0], CF, PHI, true);
  __syncthreads();
}

// MG[r][h] = PSI[r][h] * V[r][h] (vstride 0: the one row V broadcast over the tile).
__device__ __forceinline__ void merge(float *MG, const float *PSI, const float *V, int vstride,
                                      int H) {
  for (int e = threadIdx.x; e < kRows * H; e += kThreads) {
    const int r = e / H, h = e - r * H;
    MG[r * kPitch + h] = __fmul_rn(PSI[r * kPitch + h], V[r * vstride + h]);
  }
  __syncthreads();
}

// IQN's tile kernel.  Shared memory: both Q networks (trunk + head, Plan slot 0), both
// embeddings (slot 1), c-bar of each, the cosine frequencies, the gradient accumulators of the
// online network and the embedding, and the row tiles.  kWeighted: row g's gradient and loss
// are scaled by weights[g] with one multiply each, so unit weights change no bit.
template <bool kWeighted>
__device__ __forceinline__ void iqn_tile_pass(const wdb_dqn_update_args &U, const wdb_iqn_args &I,
                                              const Plan &Pg, float *partials, double *psums,
                                              const int2 *windows, const float *weights) {
  constexpr int kLanes = kThreads / kRows;     // threads per row
  extern __shared__ __align__(16) float smem[];
  __shared__ Plan P;
  __shared__ double s_h[kRows], s_q[kRows];
  __shared__ int s_a[kRows], s_best[kRows];    // the rows' actions and bootstrap actions
  if (threadIdx.x == 0) P = Pg;
  __syncthreads();
  const int tid = threadIdx.x;
  float *Wq = smem, *Wt = Wq + P.wfloats[0];
  float *We = Wt + P.wfloats[0], *Wte = We + P.wfloats[1];
  float *CB = Wte + P.wfloats[1];              // c-bar: online [0, 64), target [64, 128)
  float *FQ = CB + 2 * kMaxWidth;              // cosine frequencies float(pi * c)
  float *G = FQ + kMaxWidth;                   // online network's gradients, then the embedding's
  float *Ge = G + P.gfloats[0];
  const int g_total = P.gfloats[0] + P.gfloats[1];
  float *X = G + ((g_total + 3) / 4) * 4;      // obs at slot(0)
  float *XB = X + kTile;                       // bootstrap obs at slot(n_step), then T_j
  float *CF = XB + kTile;                      // cosine features of a tile of levels
  float *PHI = CF + kTile;                     // their embedding
  float *MG = PHI + kTile;                     // psi * phi (the head's input)
  float *Z = MG + kTile;                       // head outputs, then the head delta
  float *TH = Z + kTile;                       // theta_i, then d loss / d theta_i
  float *PT = TH + kTile;                      // target psi(obs'), then d psi
  float *D0 = PT + kTile, *D1 = D0 + kTile;    // scratch and deltas
  float *H = D1 + kTile;                       // online hidden outputs on obs
  float *T = XB, *DPSI = PT;

  const int F = U.obs_dim, A = U.n_actions, L = P.L[0], ns = U.n_step;
  const int n_cos = I.n_cos, N = I.n_tau, NP = I.n_tau_prime, K = I.n_quantile_samples;
  const int NT = N + NP, Hw = P.out[1][0];
  const int hl = P.woff[0][L - 1], hpw = P.pw[0][L - 1];   // the head in the Q networks' block
  load_net(Wq, U.q, P, 0);
  load_net(Wt, U.target_q, P, 0);
  load_net(We, I.embed, P, 1);
  load_net(Wte, I.target_embed, P, 1);
  for (int c = tid; c < kMaxWidth; c += kThreads) {
    FQ[c] = (float)(3.14159265358979323846 * (double)c);
    CB[c] = 0.0f;
    CB[kMaxWidth + c] = 0.0f;
  }
  for (int e = tid; e < g_total; e += kThreads) G[e] = 0.0f;
  for (int e = tid; e < P.n_buf * kTile; e += kThreads) X[e] = 0.0f;
  __syncthreads();

  // ---- c-bar = mean_k phi(tau~_k), tau~_k = (2k + 1) / (2K), of the online and the target
  // embedding: thread h sums its column over the levels in order
  for (int net = 0; net < 2; net++) {
    float *cb = CB + net * kMaxWidth;
    for (int k0 = 0; k0 < K; k0 += kRows) {
      cos_features(CF, FQ, n_cos, [&](int r) {
        return k0 + r < K ? (float)(2 * (k0 + r) + 1) / (float)(2 * K) : 0.0f;
      });
      __syncthreads();
      embed(net == 0 ? We : Wte, P, CF, PHI);
      if (tid < Hw)
        for (int r = 0; r < kRows && k0 + r < K; r++)
          cb[tid] = __fadd_rn(cb[tid], PHI[r * kPitch + tid]);
      __syncthreads();
    }
    if (tid < Hw) cb[tid] = __fdiv_rn(cb[tid], (float)K);
  }
  __syncthreads();

  const SampledRows rows = {windows, U.capacity};
  const long long EN = P.EN, M = P.M, E = U.n_envs, Np = U.n_agents;
  const float gamma = U.gamma, kappa = U.huber_delta;
  // d loss / d theta_i = -(1 / (kappa N' B)) sum_j |tau_i - 1{u_ij < 0}| clamp(u_ij, -kappa, kappa)
  const float norm = (float)(1.0 / ((double)kappa * (double)NP * (double)M));
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
    const float *psi = H + (L - 2) * kTile;
    trunk_forward(Wq, P, 0, X, [&](int l) { return H + l * kTile; });
    trunk_forward(Wt, P, 0, XB, [&](int l) { return l == L - 2 ? PT : (l % 2 == 0 ? D0 : D1); });
    // ---- a*: the first argmax of the collapsed head on online(obs') (double_q) or target(obs')
    if (U.double_q) {
      trunk_forward(Wq, P, 0, XB, [&](int l) { return l == L - 2 ? MG : (l % 2 == 0 ? D0 : D1); });
      merge(MG, MG, CB, 0, Hw);
    } else {
      merge(MG, PT, CB + kMaxWidth, 0, Hw);
    }
    layer_forward((U.double_q ? Wq : Wt) + hl, hpw, Hw, A, MG, Z, false);
    __syncthreads();
    if (tid < kRows) {
      const long long g = g0 + tid;
      int a = -1, best = 0;
      if (g < M) {
        const Row w = rows.at(g);
        a = U.actions[(long long)rows.slot(w, 0) * EN + w.n];
        const float *z = Z + tid * kPitch;
        for (int c = 1; c < A; c++)
          if (z[best] < z[c]) best = c;
      }
      // (an action outside [0, A) -- never written by the samplers -- contributes nothing)
      s_a[tid] = a >= 0 && a < A ? a : -1;
      s_best[tid] = best;
    }
    __syncthreads();
    auto tau_of = [&](int rr, int col) {
      const long long g = g0 + rr;
      return g < M ? I.taus[g * NT + col] : 0.0f;
    };
    // ---- the target pairs: target(obs')[a*] at tau'_j into T[r][j]
    for (int j = 0; j < NP; j++) {
      cos_features(CF, FQ, n_cos, [&](int rr) { return tau_of(rr, N + j); });
      __syncthreads();
      embed(Wte, P, CF, PHI);
      merge(MG, PT, PHI, kPitch, Hw);
      layer_forward(Wt + hl, hpw, Hw, A, MG, Z, false);
      __syncthreads();
      if (tid < kRows) T[tid * kPitch + j] = Z[tid * kPitch + s_best[tid]];
    }
    __syncthreads();
    // ---- T_j: DQN's n-step recursion on each (the row's lanes, j = k, k + kLanes, ...)
    const long long g = g0 + r;
    if (g < M) {
      const Row w = rows.at(g);
      const long long env = w.n / Np;
      for (int j = k; j < NP; j += kLanes) {
        float ret = T[r * kPitch + j];
        for (int t = ns - 1; t >= 0; t--) {
          const int pk = rows.slot(w, t);
          const float om = U.done[(long long)pk * E + env] != 0 ? 0.0f : 1.0f;
          ret = __fadd_rn(__fmul_rn(__fmul_rn(om, gamma), ret),
                          U.rewards[(long long)pk * EN + w.n]);
        }
        T[r * kPitch + j] = ret;
      }
    }
    // ---- the online pairs: theta_i = online(obs)[a] at tau_i into TH[r][i]
    for (int i = 0; i < N; i++) {
      cos_features(CF, FQ, n_cos, [&](int rr) { return tau_of(rr, i); });
      __syncthreads();
      embed(We, P, CF, PHI);
      merge(MG, psi, PHI, kPitch, Hw);
      layer_forward(Wq + hl, hpw, Hw, A, MG, Z, false);
      __syncthreads();
      if (tid < kRows) TH[tid * kPitch + i] = s_a[tid] >= 0 ? Z[tid * kPitch + s_a[tid]] : 0.0f;
    }
    __syncthreads();
    const int a = s_a[r];
    if (k == 0 && g < M) {                     // the row's mean quantile and mean target
      double rbar = 0.0;
      for (int j = 0; j < NP; j++) rbar += (double)T[r * kPitch + j];
      rbar /= (double)NP;
      if (U.returns) U.returns[g] = (float)rbar;
      if (a >= 0) {
        double qbar = 0.0;
        for (int i = 0; i < N; i++) qbar += (double)TH[r * kPitch + i];
        qbar /= (double)N;
        q_acc += qbar;
        if (U.q_values) U.q_values[g] = (float)qbar;
      }
    }
    __syncthreads();
    // ---- the pairs: thread k, levels i = k, k + kLanes, ...; T_j in order; TH[r][i] becomes
    // d loss / d theta_i
    if (g < M && a >= 0) {
      const float *Tr = T + r * kPitch;
      const float wg = kWeighted ? weights[g] : 1.0f;
      double h_row = 0.0;
      for (int i = k; i < N; i += kLanes) {
        const float th = TH[r * kPitch + i];
        const float tau = I.taus[g * NT + i];
        float acc = 0.0f;
        for (int j = 0; j < NP; j++) {
          const float u = __fsub_rn(Tr[j], th);
          const float m = u < 0.0f ? __fsub_rn(1.0f, tau) : tau;     // |tau - 1{u < 0}|
          acc = fmaf(m, fminf(fmaxf(u, -kappa), kappa), acc);
          const double au = fabs((double)u);
          h_row += (double)m * (au < (double)kappa ? 0.5 * au * au
                                                   : (double)kappa * (au - 0.5 * (double)kappa));
        }
        if constexpr (kWeighted) acc = __fmul_rn(acc, wg);
        TH[r * kPitch + i] = __fmul_rn(-acc, norm);
      }
      if constexpr (kWeighted) h_row *= (double)wg;
      h_acc += h_row;
    }
    __syncthreads();
    // ---- backward over the online pairs, the embedding recomputed: the head gradient on
    // psi * phi, d merge = W^T dz, d psi += d merge * phi (i in order), d phi = d merge * psi
    // through the ReLU into the embedding's gradient on the cosine features
    for (int i = 0; i < N; i++) {
      cos_features(CF, FQ, n_cos, [&](int rr) { return tau_of(rr, i); });
      __syncthreads();
      embed(We, P, CF, PHI);
      for (int e = tid; e < kRows * Hw; e += kThreads) {
        const int rr = e / Hw, h = e - rr * Hw;
        MG[rr * kPitch + h] = __fmul_rn(psi[rr * kPitch + h], PHI[rr * kPitch + h]);
      }
      for (int e = tid; e < kRows * A; e += kThreads) {
        const int rr = e / A, c = e - rr * A;
        Z[rr * kPitch + c] = c == s_a[rr] ? TH[rr * kPitch + i] : 0.0f;
      }
      __syncthreads();
      layer_grad(G + P.goff[0][L - 1], Hw, A, Z, MG);
      layer_backward(Wq + hl, hpw, Hw, A, Z, D0, nullptr, 0);
      __syncthreads();
      for (int e = tid; e < kRows * Hw; e += kThreads) {
        const int rr = e / Hw, h = e - rr * Hw, at = rr * kPitch + h;
        const float dm = D0[at], phi = PHI[at];
        DPSI[at] = i == 0 ? __fmul_rn(dm, phi) : fmaf(dm, phi, DPSI[at]);
        D1[at] = phi > 0.0f ? __fmul_rn(dm, psi[at]) : 0.0f;
      }
      __syncthreads();
      layer_grad(Ge, n_cos, Hw, D1, CF);
      __syncthreads();
    }
    // ---- d psi through the trunk's last ReLU, then back through the trunk
    for (int e = tid; e < kRows * Hw; e += kThreads) {
      const int at = (e / Hw) * kPitch + e % Hw;
      if (!(psi[at] > 0.0f)) DPSI[at] = 0.0f;
    }
    __syncthreads();
    const float *d = DPSI;
    float *nxt = D0;
    for (int l = L - 2; l >= 0; l--) {
      const float *x = l == 0 ? X : H + (l - 1) * kTile;
      layer_grad(G + P.goff[0][l], P.in[0][l], P.out[0][l], d, x);
      if (l > 0)
        layer_backward(Wq + P.woff[0][l], P.pw[0][l], P.in[0][l], P.out[0][l], d, nxt, x, 0);
      __syncthreads();
      d = nxt;
      nxt = nxt == D0 ? D1 : D0;
    }
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
    psums[2 * blockIdx.x] = a / ((double)kappa * (double)NP);
    psums[2 * blockIdx.x + 1] = b;
  }
}

__global__ void __launch_bounds__(kThreads, 1)
iqn_kernel(const __grid_constant__ wdb_dqn_update_args U, const __grid_constant__ wdb_iqn_args I,
           const __grid_constant__ Plan Pg, float *partials, double *psums, const int2 *windows) {
  iqn_tile_pass<false>(U, I, Pg, partials, psums, windows, nullptr);
}

__global__ void __launch_bounds__(kThreads, 1)
iqn_prioritized_kernel(const __grid_constant__ wdb_dqn_update_args U,
                       const __grid_constant__ wdb_iqn_args I, const __grid_constant__ Plan Pg,
                       float *partials, double *psums, const int2 *windows,
                       const float *weights) {
  iqn_tile_pass<true>(U, I, Pg, partials, psums, windows, weights);
}

// IQN's plan: DQN's Q networks (at least one hidden layer) in the actor-shaped slot and the
// tau embedding Linear(n_cos, H) in the critic-shaped one, H the trunk's width.  The kernel
// holds both Q networks and both embeddings, c-bar of each and the cosine frequencies, both
// gradient blocks and 10 + (hidden layers) row tiles.
bool iqn_plan(const wdb_dqn_update_args *u, const wdb_iqn_args *q, const wdb_replay_windows *w,
              Plan *p) {
  if (!u || !q || !w || !(u->huber_delta > 0.0f)) return false;
  if (q->n_cos < 1 || q->n_cos > kMaxWidth || q->n_tau < 1 || q->n_tau > kMaxWidth ||
      q->n_tau_prime < 1 || q->n_tau_prime > kMaxWidth || q->n_quantile_samples < 1 ||
      q->n_quantile_samples > kMaxQuantileSamples)
    return false;
  if (u->n_actions < 1 || u->q.n_hidden < 1) return false;
  const wdb_ddpg_net *qs[2] = {&u->q, &u->target_q};
  const wdb_ddpg_net *const *nets[2] = {qs, qs};
  const int count[2] = {2, 2};
  if (!plan_layout(u->n_envs, u->n_agents, u->obs_dim, 1, u->n_actions, u->capacity, 0,
                   u->n_step, w, nets, count, p))
    return false;
  const int H = p->out[0][p->L[0] - 2];
  int pw = round_up(q->n_cos, 4);
  if (pw % 8 == 0) pw += 4;                    // as plan_layout pitches a weight row
  p->L[1] = 1;
  p->in[1][0] = q->n_cos;
  p->out[1][0] = H;
  p->pw[1][0] = pw;
  p->woff[1][0] = 0;
  p->goff[1][0] = 0;
  p->wfloats[1] = round_up(H * pw + H, 4);
  p->gfloats[1] = H * q->n_cos + H;
  return plan_smem(p, 10 + (p->L[0] - 1), 2ll * (p->wfloats[0] + p->wfloats[1]) + 3 * kMaxWidth,
                   p->gfloats[0] + p->gfloats[1]);
}

// weights NULL: the uniform-replay kernel; else the importance-weighted one.
int iqn_update_sampled(void *stream, const wdb_dqn_update_args *u, const wdb_iqn_args *q,
                       const wdb_replay_windows *w, const float *weights) {
  Plan P;
  if (!iqn_plan(u, q, w, &P)) return (int)cudaErrorInvalidValue;
  if (!q->taus || !net_ok(q->embed, 1, true) || !net_ok(q->target_embed, 1, false))
    return (int)cudaErrorInvalidValue;
  static size_t configured[2] = {0, 0};
  return launch_q_pass(stream, u, P, w, weights, configured, &q->embed, iqn_kernel,
                       iqn_prioritized_kernel, *u, *q, P);
}

}  // namespace

// ---------------------------------------------------------------------------- entry points
// IQN: DQN's argument struct, plus the sample counts, the levels and the tau embeddings
WDB_API int wdb_iqn_update_sampled_supported(const wdb_dqn_update_args *u, const wdb_iqn_args *iqn,
                                             int n_windows) {
  const wdb_replay_windows w = {nullptr, n_windows};
  Plan P;
  return iqn_plan(u, iqn, &w, &P) ? 1 : 0;
}
WDB_API long long wdb_iqn_update_sampled_workspace_bytes(const wdb_dqn_update_args *u,
                                                         const wdb_iqn_args *iqn, int n_windows) {
  const wdb_replay_windows w = {nullptr, n_windows};
  Plan P;
  return iqn_plan(u, iqn, &w, &P) ? workspace_bytes(P) : -1;
}
WDB_API int wdb_iqn_update_sampled(void *stream, const wdb_dqn_update_args *u,
                                   const wdb_iqn_args *iqn, const wdb_replay_windows *w,
                                   const float *weights) {
  return iqn_update_sampled(stream, u, iqn, w, weights);
}
