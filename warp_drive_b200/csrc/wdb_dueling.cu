// wdb_dueling.cu -- the dueling head's fold into a plain MLP head and the unfold of its gradients
// (include/wdb200.h, wdb_dueling_*).
//
// A dueling head (Wang et al. 2016, mean combine) is linear in its output layers, so it is
// exactly a plain head over the stacked stream hidden layers: the DQN and C51 update passes and
// the one-launch rollout run it as such.  The fold writes the folded layers from the stream
// parameters before a pass; the unfold maps the folded layers' gradients back onto the stream
// parameters after it (the transpose of the fold).  Each is one launch of one element per
// thread; every mean over actions is a float32 sum over c = 0 .. A - 1 in order, divided by A.
#include "wdb_common.cuh"

using namespace wdb;

namespace {

constexpr int kThreads = 256;
constexpr long long kMaxBlocks = 4096;

// x[a N + j][k] - (1/A) sum_c x[c N + j][k] of a row-major [A N, ld] block.
__device__ __forceinline__ float centered(const float *x, long long ld, int A, int N, int a, int j,
                                          long long k) {
  float s = 0.0f;
  for (int c = 0; c < A; ++c) s += x[(long long)(c * N + j) * ld + k];
  return x[(long long)(a * N + j) * ld + k] - s / (float)A;
}

// The element counts of the folded layers: hidden weight, hidden bias, output weight, output bias.
struct Folded {
  long long hw, hb, ow, ob;
  __host__ __device__ long long total() const { return hw + hb + ow + ob; }
};

__host__ __device__ inline Folded folded_sizes(const wdb_dueling_head &h) {
  const long long S = h.stream_dim, AN = (long long)h.n_actions * h.n_atoms;
  const long long K = S > 0 ? 2 * S : h.in_dim;
  return {2 * S * h.in_dim, 2 * S, AN * K, AN};
}

// The element counts of the stream gradients, in the unfold's order.
struct Streams {
  long long hw, hb, vow, vob, aow, aob;
  __host__ __device__ long long total() const { return 2 * (hw + hb) + vow + vob + aow + aob; }
};

__host__ __device__ inline Streams stream_sizes(const wdb_dueling_head &h) {
  const long long S = h.stream_dim, N = h.n_atoms, AN = (long long)h.n_actions * N;
  const long long Kin = S > 0 ? S : h.in_dim;
  return {S * h.in_dim, S, N * Kin, N, AN * Kin, AN};
}

__device__ void fold_element(const wdb_dueling_head &h, const Folded &f, long long i) {
  const int A = h.n_actions, N = h.n_atoms, S = h.stream_dim, H = h.in_dim;
  if (i < f.hw) {                                  // stacked hidden weights [2S, H]
    const long long row = i / H, k = i % H;
    h.hw[i] = row < S ? h.value_hw[row * H + k] : h.adv_hw[(row - S) * H + k];
    return;
  }
  i -= f.hw;
  if (i < f.hb) {
    h.hb[i] = i < S ? h.value_hb[i] : h.adv_hb[i - S];
    return;
  }
  i -= f.hb;
  if (i < f.ow) {                                  // output weights [A N, K]
    const long long K = S > 0 ? 2 * S : H;
    const long long r = i / K, k = i % K;
    const int a = (int)(r / N), j = (int)(r % N);
    if (S == 0)
      h.ow[i] = h.value_ow[j * (long long)H + k] + centered(h.adv_ow, H, A, N, a, j, k);
    else if (k < S)
      h.ow[i] = h.value_ow[j * (long long)S + k];
    else
      h.ow[i] = centered(h.adv_ow, S, A, N, a, j, k - S);
    return;
  }
  i -= f.ow;
  const int a = (int)(i / N), j = (int)(i % N);   // output bias [A N]
  h.ob[i] = h.value_ob[j] + centered(h.adv_ob, 1, A, N, a, j, 0);
}

__global__ void __launch_bounds__(kThreads)
dueling_fold_kernel(wdb_dueling_head online, wdb_dueling_head target) {
  const wdb_dueling_head &h = blockIdx.y == 0 ? online : target;
  const Folded f = folded_sizes(h);
  const long long total = f.total();
  for (long long i = (long long)blockIdx.x * kThreads + threadIdx.x; i < total;
       i += (long long)gridDim.x * kThreads)
    fold_element(h, f, i);
}

__device__ void unfold_element(const wdb_dueling_head &h, const Streams &s, long long i) {
  const int A = h.n_actions, N = h.n_atoms, S = h.stream_dim, H = h.in_dim;
  if (i < 2 * s.hw) {                              // hidden weights: rows of ghw [2S, H]
    if (i < s.hw) h.value_ghw[i] = h.ghw[i];
    else h.adv_ghw[i - s.hw] = h.ghw[i];
    return;
  }
  i -= 2 * s.hw;
  if (i < 2 * s.hb) {
    if (i < s.hb) h.value_ghb[i] = h.ghb[i];
    else h.adv_ghb[i - s.hb] = h.ghb[i];
    return;
  }
  i -= 2 * s.hb;
  const long long Kin = S > 0 ? S : H, K = S > 0 ? 2 * S : H;
  if (i < s.vow) {                                 // value output [N, Kin]: sum over actions
    const long long j = i / Kin, k = i % Kin;
    float acc = 0.0f;
    for (int a = 0; a < A; ++a) acc += h.gow[(a * N + j) * K + k];
    h.value_gow[i] = acc;
    return;
  }
  i -= s.vow;
  if (i < s.vob) {
    float acc = 0.0f;
    for (int a = 0; a < A; ++a) acc += h.gob[a * N + i];
    h.value_gob[i] = acc;
    return;
  }
  i -= s.vob;
  if (i < s.aow) {                                 // advantage output [A N, Kin]: centred
    const long long r = i / Kin, k = i % Kin;
    h.adv_gow[i] = centered(h.gow, K, A, N, (int)(r / N), (int)(r % N), k + (S > 0 ? S : 0));
    return;
  }
  i -= s.aow;
  h.adv_gob[i] = centered(h.gob, 1, A, N, (int)(i / N), (int)(i % N), 0);
}

__global__ void __launch_bounds__(kThreads) dueling_unfold_kernel(wdb_dueling_head h) {
  const Streams s = stream_sizes(h);
  const long long total = s.total();
  for (long long i = (long long)blockIdx.x * kThreads + threadIdx.x; i < total;
       i += (long long)gridDim.x * kThreads)
    unfold_element(h, s, i);
}

bool shape_ok(const wdb_dueling_head *h) {
  if (!h || h->n_actions < 1 || h->n_atoms < 1 || h->in_dim < 1 || h->stream_dim < 0) return false;
  const long long lim = 1ll << 31;
  if ((long long)h->n_actions * h->n_atoms >= lim) return false;
  const Folded f = folded_sizes(*h);
  const Streams s = stream_sizes(*h);
  return f.hw < lim && f.ow < lim && s.aow < lim;
}

bool fold_pointers_ok(const wdb_dueling_head *h) {
  if (!h->value_ow || !h->value_ob || !h->adv_ow || !h->adv_ob || !h->ow || !h->ob) return false;
  if (h->stream_dim > 0 && (!h->value_hw || !h->value_hb || !h->adv_hw || !h->adv_hb || !h->hw ||
                            !h->hb))
    return false;
  return true;
}

unsigned blocks_for(long long total) {
  const long long b = (total + kThreads - 1) / kThreads;
  return (unsigned)(b < 1 ? 1 : b > kMaxBlocks ? kMaxBlocks : b);
}

}  // namespace

WDB_API int wdb_dueling_fold_supported(const wdb_dueling_head *head) { return shape_ok(head); }

WDB_API int wdb_dueling_unfold_grads_supported(const wdb_dueling_head *head) {
  return shape_ok(head);
}

WDB_API int wdb_dueling_fold(void *stream, const wdb_dueling_head *head,
                             const wdb_dueling_head *target) {
  if (!shape_ok(head) || !fold_pointers_ok(head)) return (int)cudaErrorInvalidValue;
  if (target) {
    if (target->n_actions != head->n_actions || target->n_atoms != head->n_atoms ||
        target->in_dim != head->in_dim || target->stream_dim != head->stream_dim)
      return (int)cudaErrorInvalidValue;
    if (!fold_pointers_ok(target)) return (int)cudaErrorInvalidValue;
  }
  const dim3 grid(blocks_for(folded_sizes(*head).total()), target ? 2 : 1);
  dueling_fold_kernel<<<grid, kThreads, 0, as_stream(stream)>>>(*head, target ? *target : *head);
  return finish_launch();
}

WDB_API int wdb_dueling_unfold_grads(void *stream, const wdb_dueling_head *head) {
  if (!shape_ok(head)) return (int)cudaErrorInvalidValue;
  const wdb_dueling_head *h = head;
  if (!h->value_gow || !h->value_gob || !h->adv_gow || !h->adv_gob || !h->gow || !h->gob)
    return (int)cudaErrorInvalidValue;
  if (h->stream_dim > 0 && (!h->value_ghw || !h->value_ghb || !h->adv_ghw || !h->adv_ghb ||
                            !h->ghw || !h->ghb))
    return (int)cudaErrorInvalidValue;
  dueling_unfold_kernel<<<blocks_for(stream_sizes(*head).total()), kThreads, 0,
                          as_stream(stream)>>>(*head);
  return finish_launch();
}
