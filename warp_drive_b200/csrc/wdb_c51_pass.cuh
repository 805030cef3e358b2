// wdb_c51_pass.cuh -- C51's replay-update tile body, its head-block primitives and its plan,
// shared by wdb_c51_update.cu (c51_kernel, c51_prioritized_kernel) and wdb_masked_q.cu (the
// action-masked kernels).  kMasked = false is the code the pinned kernels were compiled from;
// the masked choice of a* sits under `if constexpr`.
#pragma once

#include "wdb_common.cuh"
#include "wdb_update_tiles.cuh"

namespace {

using namespace wdb;

constexpr int kLanes = kThreads / kRows;       // threads per loss row

// Shared-memory floats of one head block: N weight rows of pitch pw, then the N biases.
__host__ __device__ __forceinline__ int block_floats(int N, int pw) {
  return (N * pw + N + 3) / 4 * 4;
}

// load_net for a C51 network: the trunk as load_net lays it out, then the head as A blocks of
// N rows (block_floats apart), each a Linear of its own.
__device__ void load_c51_net(float *dst, const wdb_ddpg_net &net, const Plan &P, int N) {
  const int L = P.L[0];
  for (int l = 0; l < L; l++) {
    const int in = P.in[0][l], out = P.out[0][l], pw = P.pw[0][l];
    const int bw = block_floats(N, pw);
    const bool head = l == L - 1;
    float *W = dst + P.woff[0][l];
    const float *w = net.w[l], *b = net.b[l];
    for (int e = threadIdx.x; e < out * pw; e += kThreads) {
      const int j = e / pw, i = e - j * pw;
      W[head ? (j / N) * bw + (j % N) * pw + i : e] = i < in ? w[j * in + i] : 0.0f;
    }
    for (int j = threadIdx.x; j < out; j += kThreads)
      W[head ? (j / N) * bw + N * pw + j % N : out * pw + j] = b[j];
  }
}

// Y[r][j] = b[j] + sum_i W[j][i] X[r][i], j < N, with W, b head block blk[r] of row r (blocks
// bw floats apart from Wh): layer_forward's operation order, so a row gets the bits
// layer_forward gives on its block.
__device__ __forceinline__ void block_forward(const float *Wh, int bw, int pw, int in, int N,
                                              const float *X, float *Y, const int *blk) {
  const int j = threadIdx.x & 63, r0 = threadIdx.x >> 6;
  if (j >= N) return;
  const float *base[4];
  float a[4] = {0.0f, 0.0f, 0.0f, 0.0f};
#pragma unroll
  for (int m = 0; m < 4; m++) base[m] = Wh + blk[r0 + 4 * m] * bw;
  int i = 0;
  for (; i + 4 <= in; i += 4) {
#pragma unroll
    for (int m = 0; m < 4; m++) {
      const float4 wv = ld4(base[m] + j * pw + i);
      const float4 x = ld4(X + (r0 + 4 * m) * kPitch + i);
      a[m] = fmaf(wv.x, x.x, a[m]);
      a[m] = fmaf(wv.y, x.y, a[m]);
      a[m] = fmaf(wv.z, x.z, a[m]);
      a[m] = fmaf(wv.w, x.w, a[m]);
    }
  }
  for (; i < in; i++) {
#pragma unroll
    for (int m = 0; m < 4; m++)
      a[m] = fmaf(base[m][j * pw + i], X[(r0 + 4 * m) * kPitch + i], a[m]);
  }
#pragma unroll
  for (int m = 0; m < 4; m++) Y[(r0 + 4 * m) * kPitch + j] = a[m] + base[m][N * pw + j];
}

// DX[r][i] = sum_j W[j][i] D[r][j] (j < N in order) for i < in, W head block blk[r] of row r,
// zeroed where mask[r][i] <= 0 (the ReLU backward).
__device__ __forceinline__ void block_backward(const float *Wh, int bw, int pw, int in, int N,
                                               const float *D, float *DX, const float *mask,
                                               const int *blk) {
  const int i = threadIdx.x & 63, r0 = threadIdx.x >> 6;
  if (i >= in) return;
  const float *base[4];
  float a[4] = {0.0f, 0.0f, 0.0f, 0.0f};
#pragma unroll
  for (int m = 0; m < 4; m++) base[m] = Wh + blk[r0 + 4 * m] * bw + i;
  for (int j = 0; j < N; j++) {
#pragma unroll
    for (int m = 0; m < 4; m++) a[m] = fmaf(base[m][j * pw], D[(r0 + 4 * m) * kPitch + j], a[m]);
  }
#pragma unroll
  for (int m = 0; m < 4; m++) {
    const int at = (r0 + 4 * m) * kPitch + i;
    DX[at] = !(mask[at] > 0.0f) ? 0.0f : a[m];
  }
}

// Over a row's kLanes threads: the lanes' values combined by an xor butterfly (every lane ends
// with the same bits: each step adds the same two operands on both sides).
__device__ __forceinline__ float lanes_sum(float v) {
  for (int off = kLanes / 2; off > 0; off /= 2) v += __shfl_xor_sync(0xffffffffu, v, off, kLanes);
  return v;
}
__device__ __forceinline__ double lanes_sum(double v) {
  for (int off = kLanes / 2; off > 0; off /= 2) v += __shfl_xor_sync(0xffffffffu, v, off, kLanes);
  return v;
}
// max_j y[j] over the row (lane k: j = k, k + kLanes, ...).
__device__ __forceinline__ float lanes_max(const float *y, int N, int k) {
  float mx = -INFINITY;
  for (int j = k; j < N; j += kLanes) mx = fmaxf(mx, y[j]);
  for (int off = kLanes / 2; off > 0; off /= 2)
    mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, off, kLanes));
  return mx;
}

// C51's tile kernel.  Shared memory: both networks (trunk, then the head blocks), the support,
// the online network's gradient accumulators (the head's in blocks of N rows and N biases) and
// the row tiles.  kWeighted: row g's gradient and loss are scaled by weights[g] with one
// multiply each, so unit weights change no bit.
// kMasked (wdb_c51_update_masked): a* is the first argmax over the valid actions of
// action_mask [C, E, Np, A] at the window's slot(n_step), which every lane of the row reads; a
// row with no valid action takes every action.  Every block's expectation is still computed
// (the lanes' shuffles are collective), only the choice skips the invalid ones, so an all-ones
// mask gives the unmasked pass's bits.
template <bool kWeighted, bool kMasked = false>
__device__ __forceinline__ void c51_tile_pass(const wdb_dqn_update_args &U, const Plan &Pg, int N,
                                              const float *support, float dz, float *partials,
                                              double *psums, const int2 *windows,
                                              const float *weights,
                                              const float *action_mask = nullptr) {
  extern __shared__ __align__(16) float smem[];
  __shared__ Plan P;
  __shared__ double s_h[kRows], s_q[kRows];
  __shared__ int s_a[kRows], s_blk[kRows], s_best[kRows];
  if (threadIdx.x == 0) P = Pg;
  __syncthreads();
  const int tid = threadIdx.x;
  float *Wq = smem, *Wt = Wq + P.wfloats[0];
  float *ZS = Wt + P.wfloats[0];               // the support z_0 .. z_{N-1}
  float *G = ZS + kMaxWidth;
  const int g_total = P.gfloats[0];
  float *X = G + ((g_total + 3) / 4) * 4;      // obs at slot(0)
  float *XB = X + kTile;                       // bootstrap obs at slot(n_step), then m_i
  float *PT = XB + kTile;                      // the chooser's, then the target's psi(obs')
  float *Z = PT + kTile;                       // block logits, Tz_j, online logits, their delta
  float *LT = Z + kTile;                       // target logits of a*, then p'_j
  float *D0 = LT + kTile, *D1 = D0 + kTile;    // deltas (the obs' forwards: scratch)
  float *H = D1 + kTile;                       // online hidden outputs on obs

  const int F = U.obs_dim, A = U.n_actions, L = P.L[0], ns = U.n_step;
  const int hl = P.woff[0][L - 1], hpw = P.pw[0][L - 1], hin = P.in[0][L - 1];
  const int bw = block_floats(N, hpw);         // head block stride in a network's block
  const int gh = P.goff[0][L - 1], gbw = N * hin + N;   // head gradient, block stride
  load_c51_net(Wq, U.q, P, N);
  load_c51_net(Wt, U.target_q, P, N);
  for (int c = tid; c < kMaxWidth; c += kThreads) ZS[c] = c < N ? support[c] : 0.0f;
  for (int e = tid; e < g_total; e += kThreads) G[e] = 0.0f;
  for (int e = tid; e < P.n_buf * kTile; e += kThreads) X[e] = 0.0f;
  __syncthreads();

  const SampledRows rows = {windows, U.capacity};
  const long long EN = P.EN, M = P.M, E = U.n_envs, Np = U.n_agents;
  const float gamma = U.gamma, z_lo = ZS[0], z_hi = ZS[N - 1];
  const float norm = (float)(1.0 / (double)M);
  const int r = tid / kLanes, k = tid - r * kLanes;
  const float *psi = L > 1 ? H + (L - 2) * kTile : X;
  const float *psib = L > 1 ? PT : XB;
  const float *Wc = U.double_q ? Wq : Wt;      // the chooser of a*
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
    trunk_forward(Wq, P, 0, X, [&](int l) { return H + l * kTile; });
    trunk_forward(Wc, P, 0, XB, [&](int l) { return l == L - 2 ? PT : (l % 2 == 0 ? D0 : D1); });
    // ---- a*: every block of the chooser at obs', its expectation Q = sum_j z_j e_j / sum_j e_j,
    // e_j = expf(y_j - max y); the first argmax (every lane of the row holds the same bits)
    const long long g = g0 + r;
    int best = kMasked ? -1 : 0;               // kMasked: -1 until the first valid action
    float best_q = 0.0f;
    const float *mk = nullptr;                 // kMasked: obs' own mask row, or NULL (none valid)
    if constexpr (kMasked) {
      if (g < M) {
        const Row wm = rows.at(g);
        mk = action_mask + ((long long)rows.slot(wm, ns) * EN + wm.n) * A;
        bool any = false;
        for (int c = 0; c < A; c++) any |= mk[c] != 0.0f;
        if (!any) mk = nullptr;
      }
    }
    for (int c = 0; c < A; c++) {
      layer_forward(Wc + hl + c * bw, hpw, hin, N, psib, Z, false);
      __syncthreads();
      const float *y = Z + r * kPitch;
      const float mx = lanes_max(y, N, k);
      float s = 0.0f, q = 0.0f;
      for (int j = k; j < N; j += kLanes) {
        const float e = expf(y[j] - mx);
        s += e;
        q = fmaf(ZS[j], e, q);
      }
      const float qc = __fdiv_rn(lanes_sum(q), lanes_sum(s));
      if constexpr (kMasked) {
        if ((!mk || mk[c] != 0.0f) && (best < 0 || best_q < qc)) {
          best_q = qc;
          best = c;
        }
      } else if (c == 0 || best_q < qc) {
        best_q = qc;
        best = c;
      }
      __syncthreads();
    }
    Row w = {0, 0};
    if (k == 0) {
      int a = -1;
      if (g < M) {
        w = rows.at(g);
        a = U.actions[(long long)rows.slot(w, 0) * EN + w.n];
      }
      // (an action outside [0, A) -- never written by the samplers -- contributes nothing)
      s_a[r] = a >= 0 && a < A ? a : -1;
      s_blk[r] = a >= 0 && a < A ? a : 0;
      s_best[r] = best;
    }
    // ---- the target's block a* at obs' (double_q: its trunk first; else PT holds it)
    if (U.double_q)
      trunk_forward(Wt, P, 0, XB, [&](int l) { return l == L - 2 ? PT : (l % 2 == 0 ? D0 : D1); });
    __syncthreads();
    block_forward(Wt + hl, bw, hpw, hin, N, psib, LT, s_best);
    __syncthreads();
    // ---- per row: p'_j = e_j / sum e (LT), Tz_j (Z), then m_i (XB)
    float *lt = LT + r * kPitch, *tz = Z + r * kPitch, *mr = XB + r * kPitch;
    {
      const float mx = lanes_max(lt, N, k);
      float s = 0.0f;
      for (int j = k; j < N; j += kLanes) {
        const float e = expf(lt[j] - mx);
        lt[j] = e;
        s += e;
      }
      s = lanes_sum(s);
      for (int j = k; j < N; j += kLanes) lt[j] = __fdiv_rn(lt[j], s);
      if (g < M) w = rows.at(g);
      const long long env = w.n / Np;
      for (int j = k; j < N; j += kLanes) {
        float ret = ZS[j];
        if (g < M)
          for (int t = ns - 1; t >= 0; t--) {
            const int pk = rows.slot(w, t);
            const float om = U.done[(long long)pk * E + env] != 0 ? 0.0f : 1.0f;
            ret = __fadd_rn(__fmul_rn(__fmul_rn(om, gamma), ret),
                            U.rewards[(long long)pk * EN + w.n]);
          }
        tz[j] = fminf(fmaxf(ret, z_lo), z_hi);
      }
    }
    __syncthreads();
    // ---- the projection: thread k, atoms i = k, k + kLanes, ...; the pairs j in order
    float sm = 0.0f;
    double rbar = 0.0;
    for (int i = k; i < N; i += kLanes) {
      const float zi = ZS[i];
      float acc = 0.0f;
      for (int j = 0; j < N; j++) {
        const float c = __fsub_rn(1.0f, __fdiv_rn(fabsf(__fsub_rn(tz[j], zi)), dz));
        acc = fmaf(fminf(fmaxf(c, 0.0f), 1.0f), lt[j], acc);
      }
      mr[i] = acc;
      sm += acc;
      rbar += (double)zi * (double)acc;
    }
    sm = lanes_sum(sm);
    rbar = lanes_sum(rbar);
    __syncthreads();
    // ---- the online block a at obs into Z; the cross-entropy and d loss / d logit_i =
    // w_g (p_i sum_k m_k - m_i) / B in place
    block_forward(Wq + hl, bw, hpw, hin, N, psi, Z, s_blk);
    __syncthreads();
    const int a = s_a[r];
    float *lo = Z + r * kPitch;
    {
      const float mx = lanes_max(lo, N, k);
      float s = 0.0f;
      for (int i = k; i < N; i += kLanes) s += expf(lo[i] - mx);
      s = lanes_sum(s);
      const double lse = (double)mx + log((double)s);
      const bool live = g < M && a >= 0;
      const float wg = kWeighted && live ? weights[g] : 1.0f;
      double h_row = 0.0, qbar = 0.0;
      for (int i = k; i < N; i += kLanes) {
        const float p = __fdiv_rn(expf(lo[i] - mx), s), m = mr[i];
        h_row += (double)m * (lse - (double)lo[i]);
        qbar += (double)ZS[i] * (double)p;
        float d = __fsub_rn(__fmul_rn(p, sm), m);
        if constexpr (kWeighted) d = __fmul_rn(d, wg);
        lo[i] = live ? __fmul_rn(d, norm) : 0.0f;
      }
      qbar = lanes_sum(qbar);
      if (live) {
        if constexpr (kWeighted) h_row *= (double)wg;
        h_acc += h_row;
      }
      if (k == 0 && g < M) {                   // the row's Q-bar and R-bar
        if (U.returns) U.returns[g] = (float)rbar;
        if (a >= 0) {
          q_acc += qbar;
          if (U.q_values) U.q_values[g] = (float)qbar;
        }
      }
    }
    __syncthreads();
    // ---- the head gradient block by block: block c's rows are the windows of action c
    for (int c = 0; c < A; c++) {
      for (int e = tid; e < kRows * N; e += kThreads) {
        const int rr = e / N, j = e - rr * N;
        D1[rr * kPitch + j] = s_a[rr] == c ? Z[rr * kPitch + j] : 0.0f;
      }
      __syncthreads();
      layer_grad(G + gh + c * gbw, hin, N, D1, psi);
      __syncthreads();
    }
    // ---- d psi through the rows' blocks and the trunk's last ReLU, then back through the trunk
    if (L > 1) {
      block_backward(Wq + hl, bw, hpw, hin, N, Z, D0, psi, s_blk);
      __syncthreads();
      const float *d = D0;
      float *nxt = D1;
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
  }

  // ---- this CTA's partials, the head's blocks back in the packed layout (W [A N, hin], then
  // b [A N]); sums[0] = sum_g w_g loss_g, sums[1] = sum_g Q-bar_g
  float *part = partials + (long long)blockIdx.x * g_total;
  for (int e = tid; e < g_total; e += kThreads) {
    int at = e;
    if (e >= gh) {
      const int c = (e - gh) / gbw, o = e - gh - c * gbw;
      at = o < N * hin ? gh + c * N * hin + o : gh + A * N * hin + c * N + (o - N * hin);
    }
    part[at] = G[e];
  }
  h_acc = lanes_sum(h_acc);
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
    psums[2 * blockIdx.x] = a;
    psums[2 * blockIdx.x + 1] = b;
  }
}

// C51's plan: DQN's Q networks in the actor-shaped slot, laid out by plan_layout with a head of
// one block (N rows), then the head widened to A blocks: A N rows in the Plan (so the gradient
// segments are the packed head's), A block_floats in each network's shared-memory block.  The
// kernel holds both networks, the support, their gradient block and 7 + (hidden layers) row
// tiles.
bool c51_plan(const wdb_dqn_update_args *u, int N, const wdb_replay_windows *w, Plan *p) {
  if (!u || !w || N < 2 || N > kMaxWidth || u->n_actions < 1 || u->n_actions > kMaxWidth)
    return false;
  const wdb_ddpg_net *qs[2] = {&u->q, &u->target_q};
  const wdb_ddpg_net *const *nets[2] = {qs, qs};
  const int count[2] = {2, 2};
  if (!plan_layout(u->n_envs, u->n_agents, u->obs_dim, 1, N, u->capacity, 0, u->n_step, w, nets,
                   count, p))
    return false;
  const int L = p->L[0], A = u->n_actions, hin = p->in[0][L - 1];
  p->out[0][L - 1] = A * N;
  p->wfloats[0] = p->woff[0][L - 1] + A * block_floats(N, p->pw[0][L - 1]);
  p->gfloats[0] = p->goff[0][L - 1] + A * N * hin + A * N;
  return plan_smem(p, 7 + (L - 1), 2ll * p->wfloats[0] + kMaxWidth, p->gfloats[0]);
}

}  // namespace
