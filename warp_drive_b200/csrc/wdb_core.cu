// wdb_core.cu -- RNG, samplers, fused done-masked reset, episode log, testkernel.
// Each kernel cites the reference kernel it replaces (paths under /root/reference).
#include "wdb_common.cuh"
#include "wdb_sa_physics.cuh"

namespace wdb {
long long g_launch_count = 0;
}

using namespace wdb;

WDB_API int wdb_abi_version(void) { return WDB_ABI_VERSION; }
WDB_API const char *wdb_error_string(int err) {
  return cudaGetErrorString(static_cast<cudaError_t>(err));
}
WDB_API long long wdb_launch_count(void) { return g_launch_count; }

// ============================================================================ RNG
WDB_API long long wdb_rng_state_bytes(long long n_streams) {
  return (long long)sizeof(RngHeader) + 8ll * n_streams;
}

// replaces init_random (core/random.cu:14-23): no device heap, one coalesced u64/stream
__global__ void rng_init_kernel(void *state, long long n_streams, unsigned long long seed) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i == 0) {
    RngHeader *h = reinterpret_cast<RngHeader *>(state);
    h->seed = seed;
    h->n_streams = (unsigned long long)n_streams;
  }
  if (i < n_streams) rng_offsets(state)[i] = 0ull;
}

WDB_API int wdb_rng_init(void *stream, void *rng_state, long long n_streams,
                         unsigned long long seed) {
  if (!rng_state || n_streams <= 0) return (int)cudaErrorInvalidValue;
  const int block = 256;
  const int grid = (int)((n_streams + block - 1) / block);
  rng_init_kernel<<<grid, block, 0, as_stream(stream)>>>(rng_state, n_streams, seed);
  return finish_launch();
}

__global__ void rng_draw_kernel(void *state, uint4 *out, long long n_streams) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_streams) return;
  const RngHeader h = *reinterpret_cast<const RngHeader *>(state);
  unsigned long long *off = rng_offsets(state);
  const unsigned long long o = off[i];
  out[i] = rng_draw4(h, (unsigned long long)i, o);
  off[i] = o + 1;
}

WDB_API int wdb_rng_draw_u32x4(void *stream, void *rng_state, unsigned int *out,
                               long long n_streams) {
  if (!rng_state || !out || n_streams <= 0) return (int)cudaErrorInvalidValue;
  const int block = 256;
  rng_draw_kernel<<<(int)((n_streams + block - 1) / block), block, 0, as_stream(stream)>>>(
      rng_state, reinterpret_cast<uint4 *>(out), n_streams);
  return finish_launch();
}

// ======================================================================== sampler
// replaces sample_actions (core/random.cu:51-85).  One thread per (env, agent) row, but
// the rows of a CTA are staged through shared memory so that the global reads of probs
// and the (optional) writes of cum_distr are fully coalesced; the reference reads and
// writes them with a stride of n_actions*4 bytes per thread.
// kNonzero: select_index_nonzero instead of the reference's search_index (masked policies).
constexpr int kSampleRows = 128;

template <bool kNonzero>
__global__ void __launch_bounds__(kSampleRows)
sample_actions_kernel(void *rng_state, const float *__restrict__ probs,
                      int *__restrict__ actions, float *__restrict__ cum_distr,
                      long long n_rows, int A, int use_argmax,
                      int *__restrict__ actions_combined, int cstride, int coffset,
                      const float *__restrict__ uniforms) {
  extern __shared__ float s_p[];  // [kSampleRows][As], As odd -> conflict-free rows
  const int As = A | 1;
  const long long row0 = (long long)blockIdx.x * kSampleRows;
  const int rows = (int)min((long long)kSampleRows, n_rows - row0);
  const float *gp = probs + row0 * A;
  for (int i = threadIdx.x; i < rows * A; i += kSampleRows)
    s_p[(i / A) * As + (i % A)] = gp[i];
  __syncthreads();

  const int r = threadIdx.x;
  if (r < rows) {
    float *p = s_p + r * As;
    const long long pos = row0 + r;
    int ind;
    if (use_argmax) {  // random.cu:58-69 (first max wins)
      float max_p = p[0];
      ind = 0;
      for (int i = 1; i < A; i++)
        if (max_p < p[i]) { max_p = p[i]; ind = i; }
    } else {
      float u;
      if (uniforms) {
        u = uniforms[pos];
      } else {
        const RngHeader h = *reinterpret_cast<const RngHeader *>(rng_state);
        unsigned long long *off = rng_offsets(rng_state);
        const unsigned long long o = off[pos];
        u = u32_to_uniform(rng_draw4(h, (unsigned long long)pos, o).x);
        off[pos] = o + 1;
      }
      if constexpr (kNonzero) {
        ind = select_index_nonzero(p, A, u);
      } else {
        float c = p[0];  // random.cu:75-80 sequential float32 CDF
        for (int i = 1; i < A; i++) { c = p[i] + c; p[i] = c; }
        ind = search_index(p, 1, u, A - 1);
      }
    }
    actions[pos] = ind;
    if (actions_combined) actions_combined[pos * cstride + coffset] = ind;
  }
  if (cum_distr && !use_argmax) {
    __syncthreads();
    float *gc = cum_distr + row0 * A;
    for (int i = threadIdx.x; i < rows * A; i += kSampleRows)
      gc[i] = s_p[(i / A) * As + (i % A)];
  }
}

template <bool kNonzero>
static int launch_sample_actions(void *stream, void *rng_state, const float *probs, int *actions,
                                 float *cum_distr, int n_envs, int n_agents, int n_actions,
                                 int use_argmax, int *actions_combined, int combined_stride,
                                 int combined_offset, const float *uniforms) {
  if (!probs || !actions || n_envs <= 0 || n_agents <= 0 || n_actions <= 0)
    return (int)cudaErrorInvalidValue;
  if (!use_argmax && !uniforms && !rng_state) return (int)cudaErrorInvalidValue;
  const long long n_rows = (long long)n_envs * n_agents;
  const int grid = (int)((n_rows + kSampleRows - 1) / kSampleRows);
  const size_t smem = sizeof(float) * kSampleRows * (size_t)(n_actions | 1);
  if (smem > 48 * 1024) {
    cudaError_t e = cudaFuncSetAttribute(sample_actions_kernel<kNonzero>,
                                         cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         (int)smem);
    if (e != cudaSuccess) return (int)e;
  }
  sample_actions_kernel<kNonzero><<<grid, kSampleRows, smem, as_stream(stream)>>>(
      rng_state, probs, actions, cum_distr, n_rows, n_actions, use_argmax,
      actions_combined, combined_stride, combined_offset, uniforms);
  return finish_launch();
}

WDB_API int wdb_sample_actions(void *stream, void *rng_state, const float *probs,
                               int *actions, float *cum_distr, int n_envs, int n_agents,
                               int n_actions, int use_argmax, int *actions_combined,
                               int combined_stride, int combined_offset,
                               const float *uniforms) {
  return launch_sample_actions<false>(stream, rng_state, probs, actions, cum_distr, n_envs,
                                      n_agents, n_actions, use_argmax, actions_combined,
                                      combined_stride, combined_offset, uniforms);
}

WDB_API int wdb_sample_actions_nonzero(void *stream, void *rng_state, const float *probs,
                                       int *actions, float *cum_distr, int n_envs, int n_agents,
                                       int n_actions, int use_argmax, int *actions_combined,
                                       int combined_stride, int combined_offset,
                                       const float *uniforms) {
  return launch_sample_actions<true>(stream, rng_state, probs, actions, cum_distr, n_envs,
                                     n_agents, n_actions, use_argmax, actions_combined,
                                     combined_stride, combined_offset, uniforms);
}

// replaces sample_ou_process (numba_includes/core/random.py:74-105); the update itself is
// ou_step (wdb_sa_physics.cuh), which the whole-rollout kernel calls as well
__global__ void sample_ou_kernel(void *rng_state, const float *__restrict__ mean,
                                 float *__restrict__ actions, float *__restrict__ ou,
                                 long long n, float damping, float stddev, float scale,
                                 const float *__restrict__ normals) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  RngHeader h = {0ull, 0ull};
  unsigned long long o = 0;
  if (rng_state && !normals) {
    h = *reinterpret_cast<const RngHeader *>(rng_state);
    o = rng_offsets(rng_state)[i];
  }
  const OuStep r = ou_step(mean[i], ou[i], normals ? normals + i : nullptr, h,
                           (unsigned long long)i, o, damping, stddev, scale);
  actions[i] = r.action;
  ou[i] = r.ou;
  if (r.draws) rng_offsets(rng_state)[i] = o + r.draws;
}

WDB_API int wdb_sample_ou_process(void *stream, void *rng_state, const float *mean,
                                  float *actions, float *ou_state, int n_envs,
                                  int n_agents, float damping, float stddev, float scale,
                                  const float *normals) {
  if (!mean || !actions || !ou_state) return (int)cudaErrorInvalidValue;
  if (!normals && !rng_state && !(scale < 1.0e-8f)) return (int)cudaErrorInvalidValue;
  const long long n = (long long)n_envs * n_agents;
  const int block = 256;
  sample_ou_kernel<<<(int)((n + block - 1) / block), block, 0, as_stream(stream)>>>(
      rng_state, mean, actions, ou_state, n, damping, stddev, scale, normals);
  return finish_launch();
}

// diagonal Gaussian policy (no reference counterpart): one thread per row, the row's math is
// gaussian_step (wdb_sa_physics.cuh), which the whole-rollout kernel calls as well
__global__ void sample_gaussian_kernel(void *rng_state, const float *__restrict__ mean,
                                       const float *__restrict__ log_std,
                                       float *__restrict__ actions, long long n_rows, int A,
                                       int use_argmax, const float *__restrict__ normals) {
  const long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n_rows) return;
  RngHeader h = {0ull, 0ull};
  unsigned long long o = 0;
  const bool draw = !use_argmax && !normals;
  if (draw) {
    h = *reinterpret_cast<const RngHeader *>(rng_state);
    o = rng_offsets(rng_state)[r];
  }
  const int draws = gaussian_step(mean + r * A, log_std, actions + r * A, A,
                                  normals ? normals + r * A : nullptr, h,
                                  (unsigned long long)r, o, use_argmax);
  if (draw) rng_offsets(rng_state)[r] = o + draws;
}

WDB_API int wdb_sample_gaussian(void *stream, void *rng_state, const float *mean,
                                const float *log_std, float *actions, long long n_rows,
                                int action_dim, int use_argmax, const float *normals) {
  if (!mean || !log_std || !actions || n_rows <= 0 || action_dim < 1)
    return (int)cudaErrorInvalidValue;
  if (!use_argmax && !normals && !rng_state) return (int)cudaErrorInvalidValue;
  const int block = 256;
  sample_gaussian_kernel<<<(int)((n_rows + block - 1) / block), block, 0, as_stream(stream)>>>(
      rng_state, mean, log_std, actions, n_rows, action_dim, use_argmax, normals);
  return finish_launch();
}

// tanh-squashed Gaussian policy (SAC's actor): one thread per row, the row's math is
// squashed_gaussian_step (wdb_sa_physics.cuh)
__global__ void sample_squashed_gaussian_kernel(void *rng_state, const float *__restrict__ head,
                                                float *__restrict__ actions, long long n_rows,
                                                int A, float scale, float bias, float lo,
                                                float hi, int use_argmax,
                                                const float *__restrict__ normals) {
  const long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n_rows) return;
  RngHeader h = {0ull, 0ull};
  unsigned long long o = 0;
  const bool draw = !use_argmax && !normals;
  if (draw) {
    h = *reinterpret_cast<const RngHeader *>(rng_state);
    o = rng_offsets(rng_state)[r];
  }
  const int draws = squashed_gaussian_step(head + r * 2 * A, actions + r * A, A, scale, bias, lo,
                                           hi, normals ? normals + r * A : nullptr, h,
                                           (unsigned long long)r, o, use_argmax);
  if (draw) rng_offsets(rng_state)[r] = o + draws;
}

WDB_API int wdb_sample_squashed_gaussian(void *stream, void *rng_state, const float *head,
                                         float *actions, long long n_rows, int action_dim,
                                         float action_scale, float action_bias,
                                         float log_std_min, float log_std_max, int use_argmax,
                                         const float *normals) {
  if (!head || !actions || n_rows <= 0 || action_dim < 1 || !(log_std_min <= log_std_max))
    return (int)cudaErrorInvalidValue;
  if (!use_argmax && !normals && !rng_state) return (int)cudaErrorInvalidValue;
  const int block = 256;
  sample_squashed_gaussian_kernel<<<(int)((n_rows + block - 1) / block), block, 0,
                                    as_stream(stream)>>>(
      rng_state, head, actions, n_rows, action_dim, action_scale, action_bias, log_std_min,
      log_std_max, use_argmax, normals);
  return finish_launch();
}

// ========================================================================== reset
// replaces reset_in_{float,int}_when_done_{2d,3d} + undo_done_flag_and_reset_timestep
// (core/reset.cu:9-75) and reset_when_done_*_from_pool (numba pool_reset.py:15-52).
// grid = (n_envs, chunks): CTA (env, c) copies the c-th slice of every registered array
// of a done env with coalesced 4-byte (16-byte when aligned) words; a not-done env costs
// one 4-byte load.  The reference's *_3d variant walks feature_dim with a stride-F
// access per thread and needs one launch per array.
__global__ void __launch_bounds__(256)
reset_when_done_kernel(const wdb_reset_desc *__restrict__ table, int n_arrays,
                       int *done, int *timestep, int force_reset, int undo,
                       void *pool_rng) {
  const int env = blockIdx.x;
  const bool hit = force_reset > 0 || done[env] > 0;
  if (!hit) return;
  unsigned long long pool_off = 0;
  RngHeader h = {0ull, 0ull};
  if (pool_rng) {
    h = *reinterpret_cast<const RngHeader *>(pool_rng);
    pool_off = rng_offsets(pool_rng)[env];
  }
  int n_pool = 0;
  for (int a = 0; a < n_arrays; a++) {
    const wdb_reset_desc d = table[a];
    const long long words = d.bytes_per_env >> 2;
    uint32_t *dst = reinterpret_cast<uint32_t *>(
        reinterpret_cast<char *>(d.dst) + (long long)env * d.bytes_per_env);
    // every thread of the env derives the same pool draw from the counter-based stream
    const long long src_row = reset_src_row(d, h, env, pool_off, n_pool);
    const uint32_t *src = reinterpret_cast<const uint32_t *>(
        reinterpret_cast<const char *>(d.ref) + src_row * d.bytes_per_env);
    const long long begin = (long long)blockIdx.y * blockDim.x + threadIdx.x;
    const long long step = (long long)gridDim.y * blockDim.x;
    if (((reinterpret_cast<uintptr_t>(dst) | reinterpret_cast<uintptr_t>(src)) & 15) == 0) {
      const long long vec = words >> 2;
      const uint4 *s4 = reinterpret_cast<const uint4 *>(src);
      uint4 *d4 = reinterpret_cast<uint4 *>(dst);
      for (long long i = begin; i < vec; i += step) d4[i] = s4[i];
      for (long long i = (vec << 2) + begin; i < words; i += step) dst[i] = src[i];
    } else {
      for (long long i = begin; i < words; i += step) dst[i] = src[i];
    }
  }
  if (pool_rng && n_pool > 0) {
    // every thread of the CTA must have read pool_off before it is advanced (a late warp
    // reading the new offset would draw a different pool row: torn reset); the early
    // return above is CTA-uniform, so the barrier is safe
    __syncthreads();
    if (blockIdx.y == 0 && threadIdx.x == 0) rng_offsets(pool_rng)[env] = pool_off + n_pool;
  }
  // undo is done by a second tiny kernel when gridDim.y > 1 (other CTAs of this env
  // still need done[env]); with gridDim.y == 1 it is safe here.
  if (undo && gridDim.y == 1) {
    __syncthreads();
    if (threadIdx.x == 0) { done[env] = 0; timestep[env] = 0; }
  }
}

// undo_done_flag_and_reset_timestep (core/reset.cu:65-75), vectorised over envs
__global__ void undo_done_kernel(int *done, int *timestep, int n_envs, int force_reset) {
  const int env = blockIdx.x * blockDim.x + threadIdx.x;
  if (env >= n_envs) return;
  if (force_reset > 0 || done[env] > 0) { done[env] = 0; timestep[env] = 0; }
}

WDB_API int wdb_reset_when_done(void *stream, const wdb_reset_desc *table_dev,
                                int n_arrays, int *done, int *timestep, int n_envs,
                                int force_reset, int undo_done_and_timestep,
                                void *pool_rng_state) {
  if (!done || !timestep || n_envs <= 0 || n_arrays < 0) return (int)cudaErrorInvalidValue;
  if (n_arrays > 0 && !table_dev) return (int)cudaErrorInvalidValue;
  int err = 0;
  // a forced reset copies every env: split each env over several CTAs to fill the GPU
  // (pool draws advance a per-env offset, so keep one CTA per env when a pool is used)
  const int chunks = (force_reset && !pool_rng_state) ? 4 : 1;
  if (n_arrays > 0) {
    dim3 grid(n_envs, chunks);
    reset_when_done_kernel<<<grid, 256, 0, as_stream(stream)>>>(
        table_dev, n_arrays, done, timestep, force_reset,
        undo_done_and_timestep && chunks == 1, pool_rng_state);
    err = finish_launch();
    if (err) return err;
  }
  if (undo_done_and_timestep && (chunks > 1 || n_arrays == 0)) {
    undo_done_kernel<<<(n_envs + 255) / 256, 256, 0, as_stream(stream)>>>(
        done, timestep, n_envs, force_reset);
    err = finish_launch();
  }
  return err;
}

// ============================================================================ log
// reset_log_mask / update_log_mask / log_one_step_in_{float,int} (core/log.cu:11-62)
__global__ void reset_log_mask_kernel(int *log_mask, int episode_length) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i <= episode_length;
       i += gridDim.x * blockDim.x)
    log_mask[i] = 0;
}

__global__ void update_log_mask_kernel(int *log_mask, int timestep, int episode_length) {
  if (threadIdx.x == 0 && blockIdx.x == 0 && timestep <= episode_length)
    log_mask[timestep] = 1;  // log.cu:22-29 (device assert on mask[t-1] dropped)
}

__global__ void log_one_step_kernel(uint32_t *log, const uint32_t *data, int n_agents,
                                    int feature_dim, int timestep, int env_id) {
  const long long per_env = (long long)n_agents * feature_dim;
  const uint32_t *src = data + (long long)env_id * per_env;
  uint32_t *dst = log + (long long)timestep * per_env;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < per_env;
       i += (long long)gridDim.x * blockDim.x)
    dst[i] = src[i];
}

WDB_API int wdb_reset_log_mask(void *stream, int *log_mask, int episode_length) {
  if (!log_mask) return (int)cudaErrorInvalidValue;
  reset_log_mask_kernel<<<1, 256, 0, as_stream(stream)>>>(log_mask, episode_length);
  return finish_launch();
}

WDB_API int wdb_update_log_mask(void *stream, int *log_mask, int timestep,
                                int episode_length) {
  if (!log_mask) return (int)cudaErrorInvalidValue;
  update_log_mask_kernel<<<1, 32, 0, as_stream(stream)>>>(log_mask, timestep, episode_length);
  return finish_launch();
}

WDB_API int wdb_log_one_step(void *stream, void *log, const void *data, int n_agents,
                             int feature_dim, int timestep, int episode_length,
                             int env_id) {
  if (!log || !data) return (int)cudaErrorInvalidValue;
  if (timestep > episode_length) return 0;  // log.cu:50 silently ignores
  const long long per_env = (long long)n_agents * feature_dim;
  const int grid = (int)min((per_env + 255) / 256, (long long)kNumSMs * 4);
  log_one_step_kernel<<<grid, 256, 0, as_stream(stream)>>>(
      reinterpret_cast<uint32_t *>(log), reinterpret_cast<const uint32_t *>(data),
      n_agents, feature_dim, timestep, env_id);
  return finish_launch();
}

// ===================================================================== testkernel
// example_envs/dummy_env/test_step.cu:9-45 (fixture for the manager tests)
__global__ void testkernel_kernel(float *x, int *y, int *done, int *actions,
                                  float multiplier, int target, int step,
                                  int episode_length, int n_agents) {
  __shared__ int reach_target;
  const int env = blockIdx.x;
  if (threadIdx.x == 0) reach_target = 0;
  __syncthreads();
  for (int agent = threadIdx.x; agent < n_agents; agent += blockDim.x) {
    const int index = env * n_agents + agent;
    x[index] = x[index] / multiplier;
    y[index] = y[index] * multiplier;
    if (y[index] >= target) atomicAdd(&reach_target, 1);
    for (int i = 0; i < 3; i++) actions[index * 3 + i] = i;
  }
  __syncthreads();
  if (threadIdx.x == 0 && (step == episode_length || reach_target > 0))
    atomicMax(&done[env], 1);
}

WDB_API int wdb_testkernel(void *stream, int n_envs, int n_agents, float *x, int *y,
                           int *done, int *actions, float multiplier, int target,
                           int step, int episode_length) {
  if (!x || !y || !done || !actions) return (int)cudaErrorInvalidValue;
  const int block = min(1024, round_up(n_agents, 32));
  testkernel_kernel<<<n_envs, block, 0, as_stream(stream)>>>(
      x, y, done, actions, multiplier, target, step, episode_length, n_agents);
  return finish_launch();
}

// ========================================================================= returns
// Bootstrapped discounted returns, backwards in time (reference: a2c.py:80-93 runs ~6
// elementwise torch kernels per timestep).  One thread per (env, agent) walks T steps;
// every step's loads/stores are unit-stride across the CTA.
__global__ void discounted_returns_kernel(const float *__restrict__ rewards,
                                          const int *__restrict__ done,
                                          const float *__restrict__ values,
                                          float *__restrict__ returns, int T, int E, int Np,
                                          float gamma) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long per_t = (long long)E * Np;
  if (i >= per_t) return;
  const int env = (int)(i / Np);
  long long idx = (long long)(T - 1) * per_t + i;
  const int d_last = done[(long long)(T - 1) * E + env] > 0;
  float ret = d_last ? rewards[idx] : values[idx];
  returns[idx] = ret;
  for (int t = T - 2; t >= 0; t--) {
    idx -= per_t;
    const int d = done[(long long)t * E + env] > 0;
    const float future = d ? 0.0f : gamma * ret;
    ret = rewards[idx] + future;
    returns[idx] = ret;
  }
}

WDB_API int wdb_discounted_returns(void *stream, const float *rewards, const int *done,
                                   const float *values, float *returns, int T, int n_envs,
                                   int n_agents, float gamma) {
  if (!rewards || !done || !values || !returns || T < 1 || n_envs < 1 || n_agents < 1)
    return (int)cudaErrorInvalidValue;
  const long long n = (long long)n_envs * n_agents;
  const int block = 128;
  discounted_returns_kernel<<<(int)((n + block - 1) / block), block, 0, as_stream(stream)>>>(
      rewards, done, values, returns, T, n_envs, n_agents, gamma);
  return finish_launch();
}

// =================================================================== replay window sampling
// windows[g] = {physical start slot, agent row} of a uniformly drawn n-step window (wdb200.h):
// Philox keyed by the seed at counter (counter, g), so the draw needs no state array and an
// update's windows are a function of (seed, counter) alone.  __umulhi(x, range) maps a 32-bit
// draw to [0, range) with each value's probability within 2^-32 of 1 / range.
__global__ void replay_sample_windows_kernel(int2 *__restrict__ windows, int n_windows,
                                             unsigned long long seed, unsigned long long counter,
                                             int oldest, int n_starts, int capacity, int n_rows) {
  const int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= n_windows) return;
  const RngHeader h = {seed, 0ull};
  const uint4 x = rng_draw4(h, (unsigned long long)g, counter);
  const int s = oldest + (int)__umulhi(x.x, (uint32_t)n_starts);
  windows[g] = make_int2(s >= capacity ? s - capacity : s, (int)__umulhi(x.y, (uint32_t)n_rows));
}

WDB_API int wdb_replay_sample_windows(void *stream, int *windows, int n_windows,
                                      unsigned long long seed, unsigned long long counter,
                                      int oldest, int filled, int capacity, int n_step,
                                      int n_rows) {
  if (!windows || n_windows < 1 || n_rows < 1 || n_step < 1 || capacity < 1)
    return (int)cudaErrorInvalidValue;
  if (filled > capacity || filled - n_step < 1 || oldest < 0 || oldest >= capacity)
    return (int)cudaErrorInvalidValue;
  const int block = 256;
  replay_sample_windows_kernel<<<(n_windows + block - 1) / block, block, 0, as_stream(stream)>>>(
      reinterpret_cast<int2 *>(windows), n_windows, seed, counter, oldest, filled - n_step,
      capacity, n_rows);
  return finish_launch();
}
