// wdb_update_tiles.cuh -- the tile primitives of the replay-update passes: the shared-memory
// Plan of a pass's networks, the row-tile layer forward / input-gradient / weight-gradient steps,
// the sampled row source and the fixed-order reduction of the per-CTA partials into the
// gradient arena, and the host launcher of the Q passes.  wdb_ddpg_update.cu (DDPG, TD3, SAC,
// DQN, QR-DQN), wdb_iqn_update.cu (IQN) and wdb_c51_update.cu (C51) build their passes on them;
// each translation unit gets its own copy (anonymous namespace).
#pragma once

#include "wdb_common.cuh"

namespace {

using namespace wdb;

constexpr int kThreads = 256;
constexpr int kRows = 16;                     // loss rows per tile
constexpr int kPitch = 68;                    // activation row pitch: float4 rows
constexpr int kTile = kRows * kPitch;         // floats of one activation buffer
constexpr int kMaxWidth = 64;
constexpr long long kMaxDynSmem = 227 * 1024 - 1024;   // the rest: the static Plan copy

struct Plan {
  int L[2];                // Linear layers (hidden + head): actor (0), critic (1)
  int in[2][4], out[2][4];
  int pw[2][4];            // smem pitch of a weight row: multiple of 4, = 4 mod 8
  int woff[2][4];          // W of layer l in the net's smem block; the bias follows W
  int wfloats[2];
  int goff[2][4];          // W gradient of layer l in the packed gradients; the bias follows
  int gfloats[2];          // actor's, critic's (the critic's start at gfloats[0])
  int n_buf;               // activation buffers
  int valid, grid;
  long long EN, M;
  long long smem_floats;
};

// The loss rows are every window of the ring (w NULL: valid * E * Np rows from `cursor`) or w's
// sampled windows (n_windows rows of n_step + 1 slots each; `cursor` is not read).
// Shape checks and the shared-memory layout of the actor shape (k = 0: F -> head, head = A, or
// 2A for SAC's mean ++ log-std) and the critic shape (k = 1: F + A -> 1).  nets[k][0] sets the
// shape; nets[k][1 .. count[k] - 1] (targets, the second critic) must have the same.
bool plan_layout(int E, int Np, int F, int A, int head, int C, int cursor, int ns,
                 const wdb_replay_windows *w, const wdb_ddpg_net *const *const nets[2],
                 const int count[2], Plan *p) {
  if (E < 1 || Np < 1 || F < 1 || A < 1 || F + A > kMaxWidth) return false;
  if (head < A || head > kMaxWidth) return false;
  if (ns < 1 || C < 2 || C < ns) return false;
  if (w ? (C < ns + 1 || w->n_windows < 1) : (cursor < 0 || cursor >= C)) return false;
  for (int k = 0; k < 2; k++) {
    const wdb_ddpg_net &n = *nets[k][0];
    if (n.n_hidden < 0 || n.n_hidden > 3) return false;
    for (int t = 1; t < count[k]; t++)
      if (nets[k][t]->n_hidden != n.n_hidden) return false;
    int prev = k == 0 ? F : F + A, woff = 0, goff = 0;
    p->L[k] = n.n_hidden + 1;
    for (int l = 0; l <= n.n_hidden; l++) {
      const int out = l < n.n_hidden ? n.widths[l] : (k == 0 ? head : 1);
      if (l < n.n_hidden) {
        if (out < 1 || out > kMaxWidth) return false;
        for (int t = 1; t < count[k]; t++)
          if (nets[k][t]->widths[l] != out) return false;
      }
      int pw = round_up(prev, 4);
      if (pw % 8 == 0) pw += 4;               // float4 rows of 8 lanes hit distinct banks
      p->in[k][l] = prev;
      p->out[k][l] = out;
      p->pw[k][l] = pw;
      p->woff[k][l] = woff;
      woff += round_up(out * pw + out, 4);
      p->goff[k][l] = goff;
      goff += out * prev + out;
      prev = out;
    }
    p->wfloats[k] = woff;
    p->gfloats[k] = goff;
  }
  p->valid = C - ns + 1;
  p->EN = (long long)E * Np;
  p->M = w ? w->n_windows : p->valid * p->EN;
  return p->M <= (1ll << 31);
}

// A kernel's activation buffers, shared-memory floats (weights, gradient accumulators, row
// tiles) and grid; false if they do not fit one CTA.
bool plan_smem(Plan *p, int n_buf, long long weight_floats, int grad_floats) {
  p->n_buf = n_buf;
  p->smem_floats = weight_floats + round_up(grad_floats, 4) + (long long)n_buf * kTile;
  if (p->smem_floats * 4 > kMaxDynSmem) return false;
  const long long tiles = (p->M + kRows - 1) / kRows;
  p->grid = (int)(tiles < kNumSMs ? tiles : kNumSMs);
  return true;
}

__device__ __forceinline__ float4 ld4(const float *p) {
  return *reinterpret_cast<const float4 *>(p);
}

// Y[r][j] = act(b[j] + sum_i W[j][i] X[r][i]) for the tile's rows; thread: column j, rows
// r0, r0 + 4, r0 + 8, r0 + 12.  Every sum runs i = 0, 1, 2, ... in order.
__device__ __forceinline__ void layer_forward(const float *W, int pw, int in, int out,
                                              const float *X, float *Y, bool relu) {
  const int j = threadIdx.x & 63, r0 = threadIdx.x >> 6;
  if (j >= out) return;
  const float *w = W + j * pw;
  float a[4] = {0.0f, 0.0f, 0.0f, 0.0f};
  int i = 0;
  for (; i + 4 <= in; i += 4) {
    const float4 wv = ld4(w + i);
#pragma unroll
    for (int m = 0; m < 4; m++) {
      const float4 x = ld4(X + (r0 + 4 * m) * kPitch + i);
      a[m] = fmaf(wv.x, x.x, a[m]);
      a[m] = fmaf(wv.y, x.y, a[m]);
      a[m] = fmaf(wv.z, x.z, a[m]);
      a[m] = fmaf(wv.w, x.w, a[m]);
    }
  }
  for (; i < in; i++) {
    const float wv = w[i];
#pragma unroll
    for (int m = 0; m < 4; m++) a[m] = fmaf(wv, X[(r0 + 4 * m) * kPitch + i], a[m]);
  }
  const float bj = W[out * pw + j];
#pragma unroll
  for (int m = 0; m < 4; m++) {
    const float y = a[m] + bj;
    Y[(r0 + 4 * m) * kPitch + j] = relu ? fmaxf(y, 0.0f) : y;
  }
}

// DX[r][i] = sum_j W[j][i] D[r][j] for columns i in [i_lo, in), zeroed where mask[r][i] <= 0
// (ReLU backward; mask = the layer's input, a ReLU output) unless mask is NULL.
__device__ __forceinline__ void layer_backward(const float *W, int pw, int in, int out,
                                               const float *D, float *DX, const float *mask,
                                               int i_lo) {
  const int i = threadIdx.x & 63, r0 = threadIdx.x >> 6;
  if (i < i_lo || i >= in) return;
  float a[4] = {0.0f, 0.0f, 0.0f, 0.0f};
  int j = 0;
  for (; j + 4 <= out; j += 4) {
    const float w0 = W[j * pw + i], w1 = W[(j + 1) * pw + i], w2 = W[(j + 2) * pw + i],
                w3 = W[(j + 3) * pw + i];
#pragma unroll
    for (int m = 0; m < 4; m++) {
      const float4 d = ld4(D + (r0 + 4 * m) * kPitch + j);
      a[m] = fmaf(w0, d.x, a[m]);
      a[m] = fmaf(w1, d.y, a[m]);
      a[m] = fmaf(w2, d.z, a[m]);
      a[m] = fmaf(w3, d.w, a[m]);
    }
  }
  for (; j < out; j++) {
    const float wv = W[j * pw + i];
#pragma unroll
    for (int m = 0; m < 4; m++) a[m] = fmaf(wv, D[(r0 + 4 * m) * kPitch + j], a[m]);
  }
#pragma unroll
  for (int m = 0; m < 4; m++) {
    const int at = (r0 + 4 * m) * kPitch + i;
    DX[at] = (mask && !(mask[at] > 0.0f)) ? 0.0f : a[m];
  }
}

// G[j][i] += sum_r D[r][j] X[r][i], G[out * in + j] += sum_r D[r][j] (the tile's rows in
// order).  Thread: column i, rows j0 .. j0 + 15 of G.  D rows are read 16 columns at a time;
// columns past `out` are in the row and never stored.
__device__ __forceinline__ void layer_grad(float *G, int in, int out, const float *D,
                                           const float *X) {
  const int i = threadIdx.x & 63, j0 = (threadIdx.x >> 6) * 16;
  if (i < in && j0 < out) {
    float acc[16];
#pragma unroll
    for (int m = 0; m < 16; m++) acc[m] = 0.0f;
    for (int r = 0; r < kRows; r++) {
      const float x = X[r * kPitch + i];
      const float *d = D + r * kPitch + j0;
#pragma unroll
      for (int q = 0; q < 4; q++) {
        const float4 dv = ld4(d + 4 * q);
        acc[4 * q + 0] = fmaf(dv.x, x, acc[4 * q + 0]);
        acc[4 * q + 1] = fmaf(dv.y, x, acc[4 * q + 1]);
        acc[4 * q + 2] = fmaf(dv.z, x, acc[4 * q + 2]);
        acc[4 * q + 3] = fmaf(dv.w, x, acc[4 * q + 3]);
      }
    }
#pragma unroll
    for (int m = 0; m < 16; m++)
      if (j0 + m < out) G[(j0 + m) * in + i] += acc[m];
  }
  if ((int)threadIdx.x < out) {
    float acc = 0.0f;
    for (int r = 0; r < kRows; r++) acc += D[r * kPitch + threadIdx.x];
    G[out * in + threadIdx.x] += acc;
  }
}

// All layers of net k on the tile; outbuf(l) is where layer l writes.
template <class OutBuf>
__device__ __forceinline__ void net_forward(const float *W, const Plan &P, int k,
                                            const float *X, OutBuf outbuf) {
  const float *x = X;
  for (int l = 0; l < P.L[k]; l++) {
    float *y = outbuf(l);
    layer_forward(W + P.woff[k][l], P.pw[k][l], P.in[k][l], P.out[k][l], x, y, l < P.L[k] - 1);
    __syncthreads();
    x = y;
  }
}

// The trunk (layers 0 .. L - 2 of net k, Linear + ReLU) on the tile; outbuf(l) is where hidden
// layer l writes.
template <class OutBuf>
__device__ __forceinline__ void trunk_forward(const float *W, const Plan &P, int k, const float *X,
                                              OutBuf outbuf) {
  const float *x = X;
  for (int l = 0; l < P.L[k] - 1; l++) {
    float *y = outbuf(l);
    layer_forward(W + P.woff[k][l], P.pw[k][l], P.in[k][l], P.out[k][l], x, y, true);
    __syncthreads();
    x = y;
  }
}

// Back-propagates the head delta Dh through net k, adding every weight gradient to G (unless
// kWeightGrads is false: G is not touched); inbuf(l) is layer l's input.  i_lo >= 0 also
// forms the input gradient of columns [i_lo, in) of layer 0; the buffer that holds it (D0 or
// D1) is returned.
template <bool kWeightGrads = true, class InBuf>
__device__ __forceinline__ const float *net_backward(const float *W, const Plan &P, int k,
                                                     float *G, const float *Dh, InBuf inbuf,
                                                     float *D0, float *D1, int i_lo) {
  const float *d = Dh;
  float *nxt = Dh == D0 ? D1 : D0;
  for (int l = P.L[k] - 1; l >= 0; l--) {
    const float *x = inbuf(l);
    if (kWeightGrads) layer_grad(G + P.goff[k][l], P.in[k][l], P.out[k][l], d, x);
    const float *Wl = W + P.woff[k][l];
    if (l > 0)
      layer_backward(Wl, P.pw[k][l], P.in[k][l], P.out[k][l], d, nxt, x, 0);
    else if (i_lo >= 0)
      layer_backward(Wl, P.pw[k][l], P.in[k][l], P.out[k][l], d, nxt, nullptr, i_lo);
    __syncthreads();
    d = nxt;
    nxt = nxt == D0 ? D1 : D0;
  }
  return d;
}

__device__ void load_net(float *dst, const wdb_ddpg_net &net, const Plan &P, int k) {
  for (int l = 0; l < P.L[k]; l++) {
    const int in = P.in[k][l], out = P.out[k][l], pw = P.pw[k][l];
    float *W = dst + P.woff[k][l];
    const float *w = net.w[l], *b = net.b[l];
    for (int e = threadIdx.x; e < out * pw; e += kThreads) {
      const int j = e / pw, i = e - j * pw;
      W[e] = i < in ? w[j * in + i] : 0.0f;
    }
    for (int j = threadIdx.x; j < out; j += kThreads) W[out * pw + j] = b[j];
  }
}

// A sampled loss row: the n-step window of agent row n (env * Np + agent) whose step 0 is at
// physical ring slot s.
struct Row {
  int s;
  long long n;
};

// The sampled row source: row g = windows[g] = {s, n}, any n_step + 1 consecutive slots (mod C)
// of the ring, in any order, duplicates allowed.  slot(w, j) is the physical slot of the
// window's step j; step n_step holds the bootstrap observation.
struct SampledRows {
  const int2 *windows;
  int C;
  __device__ __forceinline__ Row at(long long g) const {
    const int2 w = windows[g];
    return {w.x, w.y};
  }
  __device__ __forceinline__ int slot(const Row &w, int j) const {
    const int s = w.s + j;
    return s >= C ? s - C : s;
  }
};

struct Reduce {
  int grid, g_total, nseg;
  int off[16], n[16];      // segment: packed offset and length (a weight or a bias)
  float *dst[16];
};

// dst[seg][e] = sum over CTAs c = 0, 1, ... of partials[c][off[seg] + e]; sums = the same
// over the CTAs' double sums.
__global__ void ddpg_reduce_kernel(const __grid_constant__ Reduce R, const float *partials,
                                   const double *psums, double *sums) {
  const int seg = blockIdx.y;
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e < R.n[seg]) {
    const float *p = partials + R.off[seg] + e;
    float s = 0.0f;
    for (int c = 0; c < R.grid; c++) s += p[(long long)c * R.g_total];
    R.dst[seg][e] = s;
  }
  if (sums && seg == 0 && blockIdx.x == 0 && threadIdx.x == 0) {
    double a = 0.0, b = 0.0;
    for (int c = 0; c < R.grid; c++) {
      a += psums[2 * c];
      b += psums[2 * c + 1];
    }
    sums[0] = a;
    sums[1] = b;
  }
}

// ---------------------------------------------------------------------------- host side
long long workspace_bytes(const Plan &P) {
  return 16ll * P.grid + 4ll * P.grid * (P.gfloats[0] + P.gfloats[1]);
}

// Opts `kernel` into `smem` bytes of dynamic shared memory (once per size it grows to).
int allow_smem(const void *kernel, size_t smem, size_t *configured) {
  if (smem > 48 * 1024 && smem > *configured) {
    cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         (int)smem);
    if (e != cudaSuccess) return (int)e;
    *configured = smem;
  }
  return cudaSuccess;
}

// Adds the weight and bias segments of net k, packed from `base` in a CTA partial, to R.
void add_segments(Reduce *R, const Plan &P, int k, int base, const wdb_ddpg_net &net,
                  int *widest) {
  for (int l = 0; l < P.L[k]; l++) {
    const int nw = P.in[k][l] * P.out[k][l];
    R->off[R->nseg] = base + P.goff[k][l];
    R->n[R->nseg] = nw;
    R->dst[R->nseg++] = net.gw[l];
    R->off[R->nseg] = base + P.goff[k][l] + nw;
    R->n[R->nseg] = P.out[k][l];
    R->dst[R->nseg++] = net.gb[l];
    *widest = nw > *widest ? nw : *widest;
  }
}

int launch_reduce(void *stream, const Reduce &R, int widest, const float *partials,
                  const double *psums, double *sums) {
  const dim3 grid((widest + 255) / 256, R.nseg);
  ddpg_reduce_kernel<<<grid, 256, 0, as_stream(stream)>>>(R, partials, psums, sums);
  return finish_launch();
}

bool net_ok(const wdb_ddpg_net &net, int layers, bool grads) {
  for (int l = 0; l < layers; l++) {
    if (!net.w[l] || !net.b[l]) return false;
    if (grads && (!net.gw[l] || !net.gb[l])) return false;
  }
  return true;
}

// Launches one Q pass over w's sampled windows -- plain(lead..., partials, psums, windows), or
// with weights weighted(lead..., partials, psums, windows, weights), `lead` the arguments each
// kernel takes before those -- and the reduction of its per-CTA partials into the online
// network's gradients and u->sums.  embed (IQN's tau embedding, net slot 1 of P) adds its
// gradient block after the online network's.  configured: the two kernels' shared-memory
// settings (allow_smem).
template <class Plain, class Weighted, class... Lead>
int launch_q_pass(void *stream, const wdb_dqn_update_args *u, const Plan &P,
                  const wdb_replay_windows *w, const float *weights, size_t configured[2],
                  const wdb_ddpg_net *embed, Plain plain, Weighted weighted,
                  const Lead &...lead) {
  if (!w->windows || !net_ok(u->q, P.L[0], true) || !net_ok(u->target_q, P.L[0], false))
    return (int)cudaErrorInvalidValue;
  if (!u->obs || !u->actions || !u->rewards || !u->done || !u->workspace)
    return (int)cudaErrorInvalidValue;
  Reduce R = {};
  R.g_total = P.gfloats[0] + (embed ? P.gfloats[1] : 0);
  int widest = 1;
  add_segments(&R, P, 0, 0, u->q, &widest);
  if (embed) add_segments(&R, P, 1, P.gfloats[0], *embed, &widest);
  const size_t smem = (size_t)P.smem_floats * sizeof(float);
  int rc = allow_smem(weights ? (const void *)weighted : (const void *)plain, smem,
                      &configured[weights ? 1 : 0]);
  if (rc != cudaSuccess) return rc;
  double *psums = static_cast<double *>(u->workspace);
  float *partials = reinterpret_cast<float *>(psums + 2 * P.grid);
  const int2 *windows = reinterpret_cast<const int2 *>(w->windows);
  if (weights)
    weighted<<<P.grid, kThreads, smem, as_stream(stream)>>>(lead..., partials, psums, windows,
                                                            weights);
  else
    plain<<<P.grid, kThreads, smem, as_stream(stream)>>>(lead..., partials, psums, windows);
  rc = finish_launch();
  if (rc != cudaSuccess) return rc;
  R.grid = P.grid;
  return launch_reduce(stream, R, widest, partials, psums, u->sums);
}

}  // namespace
