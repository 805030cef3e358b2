// wdb_per.cu -- prioritized experience replay (Schaul et al. 2016, proportional variant) over
// the replay ring's n-step windows (include/wdb200.h, wdb_per_*).
//
// Leaves: one float32 per (physical slot s, agent row n), leaf s * n_rows + n, holding p^alpha
// of the window that starts there, or 0 while that window is not valid (it would cross the seam
// between the newest and the oldest data, or lacks its n-step look-ahead).
//
// Tree: fan-out 32 with float64 nodes, stored level by level from the parents of the leaves up
// to the root.  A node is the sum of its (up to) 32 children, padded with zeros, reduced
// pairwise: v[i] += v[i + h] for h = 16, 8, 4, 2, 1 -- one warp per node, one child per lane.
// Every write to the leaves is followed by a repair of the touched paths, one launch per level,
// each node recomputed from its children; nothing ever adds a delta, so after any history of
// writes the tree equals a fresh build from the same leaves bit for bit.  Several rows may touch
// one node: they all store the same value, computed from the level below, which the previous
// launch finished.
//
// Sampling: stratified proportional.  Row g draws u uniformly in [g S / B, (g + 1) S / B) (S:
// the root, read on the device) and descends; at each node the children are scanned in order
// with a running float64 prefix, the first child with positive mass whose prefix end exceeds u
// is entered, and u drops by the prefix before it.  When rounding puts u at or past a node's
// total, the last child with positive mass is entered: a zero-sum subtree is never entered, so
// no window of priority 0 is ever drawn.
#include "wdb_common.cuh"

using namespace wdb;

namespace {

constexpr int kFan = 32;
constexpr int kFanLog = 5;
constexpr int kMaxLevels = 8;                 // 32^7 > 2^31 leaves

// Level l = 0 are the leaves, l = 1 .. top the float64 nodes at nodes + off[l].
struct Levels {
  int top;
  long long count[kMaxLevels];
  long long off[kMaxLevels];
};

bool make_levels(long long n_leaves, Levels *L, long long *total) {
  if (n_leaves < 1 || n_leaves >= (1ll << 31)) return false;
  L->top = 0;
  L->count[0] = n_leaves;
  L->off[0] = 0;
  long long at = 0;
  do {
    const int l = ++L->top;
    L->count[l] = (L->count[l - 1] + kFan - 1) / kFan;
    L->off[l] = at;
    at += L->count[l];
  } while (L->count[L->top] > 1);
  *total = at;
  return true;
}

bool store_ok(const wdb_per_store *st, Levels *L) {
  long long total;
  if (!st || st->n_rows < 1 || st->n_step < 1 || st->capacity < st->n_step + 1) return false;
  if (!(st->alpha >= 0.0f && st->alpha <= 1.0f) || !(st->epsilon > 0.0f)) return false;
  if (!st->leaves || !st->nodes || !st->p_max) return false;
  return make_levels((long long)st->capacity * st->n_rows, L, &total);
}

__device__ __forceinline__ double child_value(const float *leaves, const double *nodes,
                                              const Levels &L, int l, long long c) {
  return l == 0 ? (double)leaves[c] : nodes[L.off[l] + c];
}

// The touched leaves of a write: the rows of `windows` (leaf windows[g].x * n_rows +
// windows[g].y, out-of-range rows skipped), or up to two leaf ranges [lo, hi).
struct Touched {
  const int2 *windows;
  int n_windows, capacity, n_rows;
  long long lo[2], hi[2];
};

// Recomputes, at level l >= 1, the node above every touched leaf: one warp per item.
__global__ void per_repair_kernel(const float *__restrict__ leaves, double *nodes,
                                  const __grid_constant__ Levels L, int l,
                                  const __grid_constant__ Touched t, long long n_items) {
  const long long item = ((long long)blockIdx.x * blockDim.x + threadIdx.x) / kWarp;
  const int lane = threadIdx.x % kWarp;
  if (item >= n_items) return;
  const int shift = kFanLog * l;
  long long node;
  if (t.windows) {
    const int2 w = t.windows[item];
    if (w.x < 0 || w.x >= t.capacity || w.y < 0 || w.y >= t.n_rows) return;
    node = ((long long)w.x * t.n_rows + w.y) >> shift;
  } else {
    const long long first = t.lo[0] >> shift, n0 = ((t.hi[0] - 1) >> shift) - first + 1;
    node = item < n0 ? first + item : (t.lo[1] >> shift) + (item - n0);
  }
  const long long c = node * kFan + lane;
  double v = c < L.count[l - 1] ? child_value(leaves, nodes, L, l - 1, c) : 0.0;
#pragma unroll
  for (int h = kFan / 2; h >= 1; h /= 2) v = __dadd_rn(v, __shfl_down_sync(0xffffffffu, v, h));
  if (lane == 0) nodes[L.off[l] + node] = v;
}

int repair(void *stream, const wdb_per_store *st, const Levels &L, const Touched &t) {
  for (int l = 1; l <= L.top; l++) {
    long long items = t.n_windows;
    if (!t.windows) {
      const int shift = kFanLog * l;
      items = 0;
      for (int r = 0; r < 2; r++)
        if (t.hi[r] > t.lo[r]) items += ((t.hi[r] - 1) >> shift) - (t.lo[r] >> shift) + 1;
    }
    if (items == 0) return cudaSuccess;
    const int block = 256;
    const long long grid = (items * kWarp + block - 1) / block;
    per_repair_kernel<<<(unsigned)grid, block, 0, as_stream(stream)>>>(st->leaves, st->nodes, L,
                                                                        l, t, items);
    const int rc = finish_launch();
    if (rc != cudaSuccess) return rc;
  }
  return cudaSuccess;
}

// ---------------------------------------------------------------------------- admit
// Slots j = 0 .. T + n_step - 1 from cursor_after - n_step - T (mod C): the first T are the
// starts that may have become valid (the previously newest n_step slots and the rollout's
// first T - n_step), the last n_step the newest slots, which now lack their look-ahead.
__global__ void per_admit_kernel(float *__restrict__ leaves, const float *__restrict__ p_max,
                                 float alpha, int C, int n_rows, int first, int T, int span,
                                 int oldest, int last_valid) {
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= (long long)span * n_rows) return;
  const int j = (int)(e / n_rows), n = (int)(e - (long long)j * n_rows);
  int s = first + j;
  s = s >= C ? s - C : s;
  float v = 0.0f;
  if (j < T) {
    int k = s - oldest;
    k = k < 0 ? k + C : k;
    if (k <= last_valid) v = powf(*p_max, alpha);
  }
  leaves[(long long)s * n_rows + n] = v;
}

// ---------------------------------------------------------------------------- sample
__device__ __forceinline__ double uniform53(uint4 x) {
  return ((double)(x.x >> 5) * 67108864.0 + (double)(x.y >> 6)) * (1.0 / 9007199254740992.0);
}

__global__ void per_sample_kernel(const float *__restrict__ leaves,
                                  const double *__restrict__ nodes, const __grid_constant__ Levels L,
                                  int n_rows, int2 *__restrict__ windows,
                                  float *__restrict__ priorities, int n_windows,
                                  unsigned long long seed, unsigned long long counter) {
  const int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= n_windows) return;
  const double S = nodes[L.off[L.top]];
  const RngHeader h = {seed, 0ull};
  const double U = uniform53(rng_draw4(h, (unsigned long long)g, counter));
  const double lo = __ddiv_rn(__dmul_rn((double)g, S), (double)n_windows);
  const double hi = __ddiv_rn(__dmul_rn((double)(g + 1), S), (double)n_windows);
  double u = __dadd_rn(lo, __dmul_rn(U, __dsub_rn(hi, lo)));
  long long node = 0;
  for (int l = L.top; l >= 1; l--) {
    const long long c0 = node * kFan;
    const long long c1 = c0 + kFan < L.count[l - 1] ? c0 + kFan : L.count[l - 1];
    long long sel = -1, last = c0;
    double prefix = 0.0, base = 0.0, last_base = 0.0;
    for (long long c = c0; c < c1; c++) {
      const double v = child_value(leaves, nodes, L, l - 1, c);
      const double next = __dadd_rn(prefix, v);
      if (v > 0.0) {
        if (sel < 0 && u < next) {
          sel = c;
          base = prefix;
        }
        last = c;
        last_base = prefix;
      }
      prefix = next;
    }
    if (sel < 0) {
      sel = last;
      base = last_base;
    }
    u = __dsub_rn(u, base);
    node = sel;
  }
  const int s = (int)(node / n_rows);
  windows[g] = make_int2(s, (int)(node - (long long)s * n_rows));
  priorities[g] = leaves[node];
}

// One CTA: the batch minimum (exact, so order-independent) and w_g = (p_g / p_min)^-beta.
__global__ void __launch_bounds__(1024) per_weights_kernel(const float *__restrict__ priorities,
                                                           float *__restrict__ weights,
                                                           int n_windows,
                                                           const float *__restrict__ beta) {
  __shared__ float s_min[kWarp];
  float m = INFINITY;
  for (int g = threadIdx.x; g < n_windows; g += blockDim.x) m = fminf(m, priorities[g]);
#pragma unroll
  for (int h = kWarp / 2; h >= 1; h /= 2) m = fminf(m, __shfl_xor_sync(0xffffffffu, m, h));
  if (threadIdx.x % kWarp == 0) s_min[threadIdx.x / kWarp] = m;
  __syncthreads();
  m = s_min[0];
  for (int k = 1; k < (int)blockDim.x / kWarp; k++) m = fminf(m, s_min[k]);
  const float nb = -*beta;
  for (int g = threadIdx.x; g < n_windows; g += blockDim.x)
    weights[g] = powf(__fdiv_rn(priorities[g], m), nb);
}

// ---------------------------------------------------------------------------- set
// Row g's window, or -1 if it is out of range or not a valid start now.
__device__ __forceinline__ long long valid_leaf(int2 w, int C, int n_rows, int oldest,
                                                int last_valid) {
  if (w.x < 0 || w.x >= C || w.y < 0 || w.y >= n_rows) return -1;
  int k = w.x - oldest;
  k = k < 0 ? k + C : k;
  return k <= last_valid ? (long long)w.x * n_rows + w.y : -1;
}

__global__ void per_clear_kernel(float *__restrict__ leaves, const int2 *__restrict__ windows,
                                 int n_windows, int C, int n_rows, int oldest, int last_valid) {
  const int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= n_windows) return;
  const long long leaf = valid_leaf(windows[g], C, n_rows, oldest, last_valid);
  if (leaf >= 0) leaves[leaf] = 0.0f;
}

// Duplicates keep the largest priority: atomicMax on the bit patterns of non-negative floats
// orders them as the floats, so the result does not depend on the order of the writes.
__global__ void per_write_kernel(float *__restrict__ leaves, float *__restrict__ p_max,
                                 const int2 *__restrict__ windows, int n_windows,
                                 const float *__restrict__ q_values,
                                 const float *__restrict__ returns, float alpha, float eps, int C,
                                 int n_rows, int oldest, int last_valid) {
  const int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= n_windows) return;
  const long long leaf = valid_leaf(windows[g], C, n_rows, oldest, last_valid);
  if (leaf < 0) return;
  float p = __fadd_rn(fabsf(__fsub_rn(q_values[g], returns[g])), eps);
  if (!(p <= 3.402823466e38f)) p = 3.402823466e38f;       // NaN / inf losses: the largest float
  atomicMax(reinterpret_cast<int *>(leaves + leaf), __float_as_int(powf(p, alpha)));
  atomicMax(reinterpret_cast<int *>(p_max), __float_as_int(p));
}

int check_windows(int n_windows, int oldest, int filled, const wdb_per_store *st) {
  if (n_windows < 1 || oldest < 0 || oldest >= st->capacity) return (int)cudaErrorInvalidValue;
  if (filled > st->capacity || filled < st->n_step + 1) return (int)cudaErrorInvalidValue;
  return cudaSuccess;
}

}  // namespace

WDB_API long long wdb_per_nodes(long long n_leaves) {
  Levels L;
  long long total;
  return make_levels(n_leaves, &L, &total) ? total : -1;
}

WDB_API int wdb_per_levels(long long n_leaves) {
  Levels L;
  long long total;
  return make_levels(n_leaves, &L, &total) ? L.top : -1;
}

WDB_API int wdb_per_admit(void *stream, const wdb_per_store *store, int cursor_before,
                          int filled_before, int cursor_after, int filled_after) {
  Levels L;
  if (!store_ok(store, &L)) return (int)cudaErrorInvalidValue;
  const int C = store->capacity, ns = store->n_step, N = store->n_rows;
  if (cursor_before < 0 || cursor_before >= C || cursor_after < 0 || cursor_after >= C)
    return (int)cudaErrorInvalidValue;
  if (filled_before < 0 || filled_before > C || filled_after > C) return (int)cudaErrorInvalidValue;
  int T = cursor_after - cursor_before;
  T = T < 0 ? T + C : T;
  // the rollout wrote T >= 1 slots (T + n_step <= C) after the data the store knew of
  if (T < 1 || T + ns > C) return (int)cudaErrorInvalidValue;
  if (filled_after != (filled_before + T < C ? filled_before + T : C))
    return (int)cudaErrorInvalidValue;
  if (filled_before < C && cursor_before != filled_before) return (int)cudaErrorInvalidValue;
  const int span = T + ns;
  int first = cursor_after - span;
  first = first < 0 ? first + C : first;
  const int oldest = filled_after == C ? cursor_after : 0;
  const long long n = (long long)span * N;
  const int block = 256;
  per_admit_kernel<<<(unsigned)((n + block - 1) / block), block, 0, as_stream(stream)>>>(
      store->leaves, store->p_max, store->alpha, C, N, first, T, span, oldest,
      filled_after - ns - 1);
  int rc = finish_launch();
  if (rc != cudaSuccess) return rc;
  Touched t = {};
  const int end = first + span;              // slots first .. end - 1, mod C
  t.lo[0] = (long long)first * N;
  t.hi[0] = (long long)(end < C ? end : C) * N;
  t.lo[1] = 0;
  t.hi[1] = end > C ? (long long)(end - C) * N : 0;
  return repair(stream, store, L, t);
}

WDB_API int wdb_per_sample_windows(void *stream, const wdb_per_store *store, int *windows,
                                   float *priorities, float *weights, int n_windows,
                                   unsigned long long seed, unsigned long long counter,
                                   const float *beta) {
  Levels L;
  if (!store_ok(store, &L) || !windows || !priorities || !weights || !beta || n_windows < 1)
    return (int)cudaErrorInvalidValue;
  const int block = 256;
  per_sample_kernel<<<(n_windows + block - 1) / block, block, 0, as_stream(stream)>>>(
      store->leaves, store->nodes, L, store->n_rows, reinterpret_cast<int2 *>(windows),
      priorities, n_windows, seed, counter);
  int rc = finish_launch();
  if (rc != cudaSuccess) return rc;
  per_weights_kernel<<<1, 1024, 0, as_stream(stream)>>>(priorities, weights, n_windows, beta);
  return finish_launch();
}

WDB_API int wdb_per_set_priorities(void *stream, const wdb_per_store *store, const int *windows,
                                   int n_windows, const float *q_values, const float *returns,
                                   int oldest, int filled) {
  Levels L;
  if (!store_ok(store, &L) || !windows || !q_values || !returns) return (int)cudaErrorInvalidValue;
  int rc = check_windows(n_windows, oldest, filled, store);
  if (rc != cudaSuccess) return rc;
  const int C = store->capacity, N = store->n_rows, last_valid = filled - store->n_step - 1;
  const int2 *w = reinterpret_cast<const int2 *>(windows);
  const int block = 256, grid = (n_windows + block - 1) / block;
  per_clear_kernel<<<grid, block, 0, as_stream(stream)>>>(store->leaves, w, n_windows, C, N,
                                                          oldest, last_valid);
  rc = finish_launch();
  if (rc != cudaSuccess) return rc;
  per_write_kernel<<<grid, block, 0, as_stream(stream)>>>(
      store->leaves, store->p_max, w, n_windows, q_values, returns, store->alpha,
      store->epsilon, C, N, oldest, last_valid);
  rc = finish_launch();
  if (rc != cudaSuccess) return rc;
  Touched t = {};
  t.windows = w;
  t.n_windows = n_windows;
  t.capacity = C;
  t.n_rows = N;
  return repair(stream, store, L, t);
}
