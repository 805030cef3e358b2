// wdb_recurrent.cu -- the per-step rollout forward of a recurrent policy (FullyConnectedGRU:
// trunk -> GRU cell -> softmax heads) and the done-masked reset of its hidden state
// (include/wdb200.h, wdb_gru_forward_bytes / wdb_gru_policy_forward / wdb_recurrent_reset_done).
//
// The forward is fp32 throughout, so the rollout acts with the numbers the fp32 training network
// computes.  Each CTA stages every weight once in shared memory (transposed, [in][out], in-dims
// padded to a multiple of 4 with zero rows) and then walks tiles of kTileRows rows (a persistent
// grid).  Every output is one thread's sum, in one fixed order:
//   acc = 0; for k = 0 .. K-1 ascending: acc = fmaf(W[j][k], x[k], acc); y = acc + b[j]
// (the zero-padded k add exact zeros).  The GRU cell is nn.GRUCell's (gate order r, z, n):
//   r  = sig(gi_r + gh_r),  z = sig(gi_z + gh_z),  n = tanhf(gi_n + r * gh_n)
//   h' = (1 - z) * n + z * h,   sig(x) = 1 / (1 + expf(-x))
// with gi = W_ih x + b_ih and gh = W_hh h + b_hh each summed as above, every other operation
// one IEEE-rounded float op (no contraction).  A head's softmax: m = max_a l_a, s = sum_a
// expf(l_a - m) ascending, p_a = expf(l_a - m) / s.  The mean head kind (FullyConnectedGaussianGRU)
// writes the logits l of its one head as they are.  The head kind is a template parameter: the
// trunk and the cell are the same code in both instantiations, so h' is the same bits, and the
// mean instantiation has no softmax.  tests/recurrent_reference.py (the mean kind:
// tests/gaussian_recurrent_reference.py) bounds every output a priori against a float64
// evaluation of the same expression.
#include <algorithm>
#include <cstddef>
#include <cstring>

#include "wdb_common.cuh"

using namespace wdb;

namespace {

constexpr int kTileRows = 16;
constexpr int kRowsPerThread = 4;
constexpr int kThreads = 256;
constexpr int kMaxIn = 256;       // observation width F
constexpr int kMaxWidth = 128;    // trunk widths and the GRU width H
constexpr int kMaxHead = 64;      // actions per head
constexpr long long kMaxSmem = 227 * 1024;

__host__ __device__ inline int pad4(int v) { return (v + 3) / 4 * 4; }

// Shared-memory layout (float offsets); every region starts on a 16-byte boundary.
struct Layout {
  int n_layers, n_heads, F, dims[2], H, heads[2];
  int in_of[4];                   // padded input width of trunk layer l, the GRU input, h
  int w_fc[2], b_fc[2], w_ih, w_hh, b_ih, b_hh, w_head[2], b_head[2];
  int x, act[2], h, gi, gh, hn, logits;
  long long floats;
};

bool make_layout(int F, int n_layers, int d0, int d1, int H, int n_heads, int a0, int a1,
                 Layout *L) {
  if (F < 1 || F > kMaxIn || n_layers < 0 || n_layers > 2 || H < 1 || H > kMaxWidth) return false;
  if (n_heads < 1 || n_heads > 2) return false;
  const int dims[2] = {d0, d1};
  for (int l = 0; l < n_layers; l++)
    if (dims[l] < 1 || dims[l] > kMaxWidth) return false;
  const int heads[2] = {a0, a1};
  for (int k = 0; k < n_heads; k++)
    if (heads[k] < 1 || heads[k] > kMaxHead) return false;
  Layout &s = *L;
  s.n_layers = n_layers;
  s.n_heads = n_heads;
  s.F = F;
  s.H = H;
  for (int l = 0; l < 2; l++) s.dims[l] = l < n_layers ? dims[l] : 0;
  for (int k = 0; k < 2; k++) s.heads[k] = k < n_heads ? heads[k] : 0;
  long long off = 0;
  auto take = [&](long long n) {
    const int at = (int)off;
    off += (n + 3) / 4 * 4;
    return at;
  };
  int in = F;
  for (int l = 0; l < n_layers; l++) {
    s.in_of[l] = pad4(in);
    s.w_fc[l] = take((long long)s.in_of[l] * dims[l]);
    s.b_fc[l] = take(dims[l]);
    in = dims[l];
  }
  const int D = in;               // the GRU's input width
  s.in_of[2] = pad4(D);
  s.in_of[3] = pad4(H);
  s.w_ih = take((long long)s.in_of[2] * 3 * H);
  s.w_hh = take((long long)s.in_of[3] * 3 * H);
  s.b_ih = take(3 * H);
  s.b_hh = take(3 * H);
  for (int k = 0; k < n_heads; k++) {
    s.w_head[k] = take((long long)s.in_of[3] * heads[k]);
    s.b_head[k] = take(heads[k]);
  }
  s.x = take((long long)kTileRows * pad4(F));
  for (int l = 0; l < n_layers; l++) s.act[l] = take((long long)kTileRows * pad4(dims[l]));
  s.h = take((long long)kTileRows * s.in_of[3]);
  s.gi = take((long long)kTileRows * 3 * H);
  s.gh = take((long long)kTileRows * 3 * H);
  s.hn = take((long long)kTileRows * s.in_of[3]);
  s.logits = take((long long)kTileRows * (s.heads[0] + s.heads[1]));
  s.floats = off;
  return off * 4 <= kMaxSmem;
}

// W [out, K] row-major (torch Linear) -> shared Wt [Kp][out], zero rows for K <= k < Kp
__device__ void stage_weight(float *dst, const float *__restrict__ W, int out, int K, int Kp) {
  for (int i = threadIdx.x; i < Kp * out; i += blockDim.x) {
    const int k = i / out, j = i - k * out;
    dst[i] = k < K ? W[(long long)j * K + k] : 0.0f;
  }
}

__device__ void stage_vector(float *dst, const float *__restrict__ v, int n) {
  for (int i = threadIdx.x; i < n; i += blockDim.x) dst[i] = v[i];
}

// dst[r][j] = (sum_k Wt[k][j] in[r][k] in ascending k, fmaf) + b[j], for r < kTileRows and
// j < out; in has row pitch Kp (a multiple of 4, zero past the real width); ReLU if asked.
__device__ void dense(const float *Wt, const float *b, const float *in, int Kp, int out,
                      float *dst, int ldo, bool relu) {
  constexpr int kGroups = kTileRows / kRowsPerThread;
  for (int o = threadIdx.x; o < out * kGroups; o += blockDim.x) {
    const int j = o % out, g = o / out;
    const float *x = in + g * kRowsPerThread * Kp;
    float acc[kRowsPerThread];
#pragma unroll
    for (int i = 0; i < kRowsPerThread; i++) acc[i] = 0.0f;
    for (int k = 0; k < Kp; k += 4) {
      const float w0 = Wt[(k + 0) * out + j], w1 = Wt[(k + 1) * out + j];
      const float w2 = Wt[(k + 2) * out + j], w3 = Wt[(k + 3) * out + j];
#pragma unroll
      for (int i = 0; i < kRowsPerThread; i++) {
        const float4 v = *reinterpret_cast<const float4 *>(x + i * Kp + k);
        acc[i] = fmaf(w0, v.x, acc[i]);
        acc[i] = fmaf(w1, v.y, acc[i]);
        acc[i] = fmaf(w2, v.z, acc[i]);
        acc[i] = fmaf(w3, v.w, acc[i]);
      }
    }
    const float bj = b[j];
#pragma unroll
    for (int i = 0; i < kRowsPerThread; i++) {
      float y = __fadd_rn(acc[i], bj);
      if (relu) y = fmaxf(y, 0.0f);
      dst[(g * kRowsPerThread + i) * ldo + j] = y;
    }
  }
}

__device__ __forceinline__ float sigmoid(float x) {
  return __fdiv_rn(1.0f, __fadd_rn(1.0f, expf(-x)));
}

// The kernel's parameter: wdb_gru_forward without its trailing head_kind, which picks the
// instantiation instead.  The parameter block keeps the layout it had before head_kind existed.
struct GruArgs {
  long long n_rows;
  int in_dim, n_layers, dims[2], hidden_size, n_heads, heads[2];
  const float *obs;
  float *hidden;
  const float *fc_weight[2], *fc_bias[2];
  const float *weight_ih, *weight_hh, *bias_ih, *bias_hh;
  const float *head_weight[2], *head_bias[2];
  float *probs[2];
};
static_assert(sizeof(GruArgs) == offsetof(wdb_gru_forward, head_kind), "GruArgs layout");
static_assert(offsetof(GruArgs, obs) == offsetof(wdb_gru_forward, obs), "GruArgs layout");
static_assert(offsetof(GruArgs, probs) == offsetof(wdb_gru_forward, probs), "GruArgs layout");

enum HeadKind { kSoftmaxHeads = 0, kMeanHead = 1 };

template <int kHeadKind>
__global__ void __launch_bounds__(kThreads, 1)
gru_policy_forward_kernel(const __grid_constant__ GruArgs args,
                          const __grid_constant__ Layout s) {
  extern __shared__ __align__(16) float sm[];
  // ---- weights, once per CTA
  int in = s.F;
  for (int l = 0; l < s.n_layers; l++) {
    stage_weight(sm + s.w_fc[l], args.fc_weight[l], s.dims[l], in, s.in_of[l]);
    stage_vector(sm + s.b_fc[l], args.fc_bias[l], s.dims[l]);
    in = s.dims[l];
  }
  const int H = s.H;
  stage_weight(sm + s.w_ih, args.weight_ih, 3 * H, in, s.in_of[2]);
  stage_weight(sm + s.w_hh, args.weight_hh, 3 * H, H, s.in_of[3]);
  stage_vector(sm + s.b_ih, args.bias_ih, 3 * H);
  stage_vector(sm + s.b_hh, args.bias_hh, 3 * H);
  for (int k = 0; k < s.n_heads; k++) {
    stage_weight(sm + s.w_head[k], args.head_weight[k], s.heads[k], H, s.in_of[3]);
    stage_vector(sm + s.b_head[k], args.head_bias[k], s.heads[k]);
  }
  // the padding columns of the activation tiles stay zero (only real columns are written)
  for (int i = threadIdx.x; i < kTileRows * s.in_of[3]; i += blockDim.x) sm[s.hn + i] = 0.0f;
  for (int l = 0; l < s.n_layers; l++)
    for (int i = threadIdx.x; i < kTileRows * pad4(s.dims[l]); i += blockDim.x)
      sm[s.act[l] + i] = 0.0f;
  __syncthreads();

  const int Fp = pad4(s.F), Hp = s.in_of[3], A_all = s.heads[0] + s.heads[1];
  const long long n_tiles = (args.n_rows + kTileRows - 1) / kTileRows;
  for (long long tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    const long long r0 = tile * kTileRows;
    const int rows = (int)min((long long)kTileRows, args.n_rows - r0);
    // ---- observations and hidden state in (zeros past the real rows and columns)
    for (int i = threadIdx.x; i < kTileRows * Fp; i += blockDim.x) {
      const int r = i / Fp, c = i - r * Fp;
      sm[s.x + i] = (r < rows && c < s.F) ? args.obs[(r0 + r) * s.F + c] : 0.0f;
    }
    for (int i = threadIdx.x; i < kTileRows * Hp; i += blockDim.x) {
      const int r = i / Hp, c = i - r * Hp;
      sm[s.h + i] = (r < rows && c < H) ? args.hidden[(r0 + r) * H + c] : 0.0f;
    }
    __syncthreads();
    // ---- trunk
    const float *x = sm + s.x;
    int xp = Fp;
    for (int l = 0; l < s.n_layers; l++) {
      const int dp = pad4(s.dims[l]);
      dense(sm + s.w_fc[l], sm + s.b_fc[l], x, xp, s.dims[l], sm + s.act[l], dp, true);
      __syncthreads();
      x = sm + s.act[l];
      xp = dp;
    }
    // ---- GRU cell
    dense(sm + s.w_ih, sm + s.b_ih, x, xp, 3 * H, sm + s.gi, 3 * H, false);
    dense(sm + s.w_hh, sm + s.b_hh, sm + s.h, Hp, 3 * H, sm + s.gh, 3 * H, false);
    __syncthreads();
    for (int i = threadIdx.x; i < kTileRows * H; i += blockDim.x) {
      const int r = i / H, c = i - r * H;
      const float *gi = sm + s.gi + r * 3 * H, *gh = sm + s.gh + r * 3 * H;
      const float rg = sigmoid(__fadd_rn(gi[c], gh[c]));
      const float zg = sigmoid(__fadd_rn(gi[H + c], gh[H + c]));
      const float ng = tanhf(__fadd_rn(gi[2 * H + c], __fmul_rn(rg, gh[2 * H + c])));
      const float hv = sm[s.h + r * Hp + c];
      const float hn = __fadd_rn(__fmul_rn(__fsub_rn(1.0f, zg), ng), __fmul_rn(zg, hv));
      sm[s.hn + r * Hp + c] = hn;
      if (r < rows) args.hidden[(r0 + r) * H + c] = hn;
    }
    __syncthreads();
    // ---- heads: logits, then one thread per (row, head) softmax, or the mean copied out
    for (int k = 0, col = 0; k < s.n_heads; col += s.heads[k], k++)
      dense(sm + s.w_head[k], sm + s.b_head[k], sm + s.hn, Hp, s.heads[k], sm + s.logits + col,
            A_all, false);
    __syncthreads();
    if constexpr (kHeadKind == kSoftmaxHeads) {
      for (int i = threadIdx.x; i < kTileRows * s.n_heads; i += blockDim.x) {
        const int r = i / s.n_heads, k = i - r * s.n_heads;
        if (r >= rows) continue;
        const int A = s.heads[k];
        const float *l = sm + s.logits + r * A_all + (k == 0 ? 0 : s.heads[0]);
        float m = l[0];
        for (int a = 1; a < A; a++) m = fmaxf(m, l[a]);
        float sum = 0.0f;
        for (int a = 0; a < A; a++) sum = __fadd_rn(sum, expf(__fsub_rn(l[a], m)));
        float *p = args.probs[k] + (r0 + r) * A;
        for (int a = 0; a < A; a++) p[a] = __fdiv_rn(expf(__fsub_rn(l[a], m)), sum);
      }
    } else {
      // one head (A_all = A): the tile's rows [rows, A] are contiguous in both places
      for (int i = threadIdx.x; i < rows * A_all; i += blockDim.x)
        args.probs[0][r0 * A_all + i] = sm[s.logits + i];
    }
    __syncthreads();
  }
}

// Grid-stride over every policy's [E, Np, H] hidden state: zero an element where done[e] > 0.
__global__ void recurrent_reset_done_kernel(const __grid_constant__ wdb_recurrent_reset table) {
  for (int p = 0; p < table.n_policies; p++) {
    const wdb_recurrent_state &st = table.policy[p];
    const long long per_env = (long long)st.n_agents * st.hidden_size;
    const long long n = per_env * table.n_envs;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n;
         i += (long long)gridDim.x * blockDim.x)
      if (table.done[i / per_env] > 0) st.hidden[i] = 0.0f;
  }
}

}  // namespace

WDB_API long long wdb_gru_forward_bytes(int in_dim, int n_layers, int d0, int d1, int hidden,
                                        int n_heads, int a0, int a1) {
  Layout L;
  return make_layout(in_dim, n_layers, d0, d1, hidden, n_heads, a0, a1, &L) ? L.floats * 4 : 0;
}

template <int kHeadKind>
static int launch_gru_forward(void *stream, const wdb_gru_forward *a, const Layout &L) {
  const int smem = (int)(L.floats * 4);
  static int configured = 0;
  if (smem > 48 * 1024 && smem > configured) {
    cudaError_t e = cudaFuncSetAttribute(gru_policy_forward_kernel<kHeadKind>,
                                         cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    if (e != cudaSuccess) return (int)e;
    configured = smem;
  }
  GruArgs k;
  std::memcpy(&k, a, sizeof(k));
  const long long n_tiles = (a->n_rows + kTileRows - 1) / kTileRows;
  const int grid = (int)(n_tiles < kNumSMs ? n_tiles : kNumSMs);
  gru_policy_forward_kernel<kHeadKind><<<grid, kThreads, smem, as_stream(stream)>>>(k, L);
  return finish_launch();
}

WDB_API int wdb_gru_policy_forward(void *stream, const wdb_gru_forward *a) {
  Layout L;
  if (!a || a->n_rows < 1 || a->n_layers < 0 || a->n_layers > 2 || a->n_heads < 1 ||
      a->n_heads > 2)
    return (int)cudaErrorInvalidValue;
  if (a->head_kind != kSoftmaxHeads && a->head_kind != kMeanHead) return (int)cudaErrorInvalidValue;
  if (a->head_kind == kMeanHead && a->n_heads != 1) return (int)cudaErrorInvalidValue;
  if (!make_layout(a->in_dim, a->n_layers, a->dims[0], a->dims[1], a->hidden_size, a->n_heads,
                   a->heads[0], a->heads[1], &L))
    return (int)cudaErrorInvalidValue;
  if (!a->obs || !a->hidden || !a->weight_ih || !a->weight_hh || !a->bias_ih || !a->bias_hh)
    return (int)cudaErrorInvalidValue;
  for (int l = 0; l < a->n_layers; l++)
    if (!a->fc_weight[l] || !a->fc_bias[l]) return (int)cudaErrorInvalidValue;
  for (int k = 0; k < a->n_heads; k++)
    if (!a->head_weight[k] || !a->head_bias[k] || !a->probs[k]) return (int)cudaErrorInvalidValue;
  return a->head_kind == kMeanHead ? launch_gru_forward<kMeanHead>(stream, a, L)
                                   : launch_gru_forward<kSoftmaxHeads>(stream, a, L);
}

WDB_API int wdb_recurrent_reset_done(void *stream, const wdb_recurrent_reset *t) {
  if (!t || !t->done || t->n_envs < 1 || t->n_policies < 1 ||
      t->n_policies > WDB_RECURRENT_MAX_POLICIES)
    return (int)cudaErrorInvalidValue;
  long long most = 0;
  for (int p = 0; p < t->n_policies; p++) {
    const wdb_recurrent_state &st = t->policy[p];
    if (!st.hidden || st.n_agents < 1 || st.hidden_size < 1) return (int)cudaErrorInvalidValue;
    most = std::max(most, (long long)st.n_agents * st.hidden_size * t->n_envs);
  }
  const int block = 256;
  const int grid = (int)std::min((most + block - 1) / block, 8LL * kNumSMs);
  recurrent_reset_done_kernel<<<grid, block, 0, as_stream(stream)>>>(*t);
  return finish_launch();
}
