// wdb_rollout_generic.cu -- the per-timestep data movement and bookkeeping of the rollout for
// ANY env (tag_gridworld, custom envs, envs with reset pools ...), i.e. for everything that
// does not have a fused step kernel of its own (SURVEY.md section 8 rows a2, a4, a6, a10).
//
// The reference does this with torch indexing per policy and per head
// (warp_drive/training/trainer_base.py:437-512 obs / action push, :514-601 reward / done push
// and the episodic sums with done_flags.nonzero() / len()): 30-40 small launches and two
// host synchronisations per timestep.  Here:
//   wdb_gather_policy_rows   [E, N, W] <-> per-policy [E, Np, W] rows, every policy in ONE
//                            launch, both directions (obs -> batch slot of each policy;
//                            per-policy probabilities -> the sampler's [E, N, A] array)
//   wdb_gather_policy_fields every key of a Dict observation (and its action mask) -> the
//                            processed observation / mask slot of each policy, ONE launch;
//                            sources may be per policy ([E, Np, ...]) and agent-last
//                            ([E, *F, Ns], transposed through shared memory)
//   wdb_rollout_bookkeep     done -> batch; per policy rewards (gather) -> batch, actions
//                            (gather) -> batch, running / episodic reward sums; step sums,
//                            completed-episode count: ONE launch, no host synchronisation;
//                            rewards / actions from the shared arrays or per-policy ones
#include "wdb_common.cuh"

using namespace wdb;

namespace {

constexpr int kGenThreads = 128;

struct GatherArgs {
  int n_envs, n_agents, width, n_policies, scatter;
  uint32_t *full;
  int np[4];
  const int *ids[4];
  uint32_t *rows[4];
  long long first_item[5];     // prefix over policies of E * Np (work items = rows)
};

// one warp per (policy, env, slot) row; lanes over the row's 4-byte elements
__global__ void __launch_bounds__(kGenThreads)
gather_rows_kernel(const __grid_constant__ GatherArgs a) {
  const int lane = threadIdx.x & 31;
  const long long warp = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (warp >= a.first_item[a.n_policies]) return;
  int p = 0;
#pragma unroll
  for (int q = 1; q < 4; q++)
    if (q < a.n_policies && warp >= a.first_item[q]) p = q;
  const long long r = warp - a.first_item[p];
  const int np = a.np[p];
  const int env = (int)(r / np), slot = (int)(r - (long long)env * np);
  const int agent = a.ids[p] ? a.ids[p][slot] : slot;
  uint32_t *f = a.full + ((long long)env * a.n_agents + agent) * a.width;
  uint32_t *q = a.rows[p] + r * a.width;
  if (a.scatter) {
    for (int i = lane; i < a.width; i += 32) f[i] = q[i];
  } else {
    for (int i = lane; i < a.width; i += 32) q[i] = f[i];
  }
}

// agent-last sources are transposed through a shared-memory tile of kTileCols columns x
// kTileAgents agents (column-major, padded by one): 32 x 32 for wide fields, narrower fields
// take more agents per tile so that a CTA still moves about kTileElems elements
constexpr int kTileElems = 1024;
constexpr int kMaxTileJobs = 4 * WDB_GATHER_MAX_FIELDS;

struct TileJob {
  int p, f;                    // policy, field
  int ta, tc;                  // agents x columns per tile (ta a multiple of 32, tc <= 32)
  int tiles_a, tiles_c;        // tiles per env along the agents / the columns
  long long first;             // first tile (CTA) of the job, counted from the tile part
};

struct FieldsArgs {
  int n_envs, n_agents, n_policies, n_fields;
  int dst_width[4][2];
  wdb_gather_field field[WDB_GATHER_MAX_FIELDS];
  int np[4];
  const int *ids[4];
  float *rows[4][2];
  long long first_item[5];     // prefix over policies of E * Np rows with an agent-first field
  long long row_blocks;        // CTAs of the row part; the tile part follows
  int n_jobs;
  TileJob job[kMaxTileJobs];
};

__host__ __device__ __forceinline__ bool feeds(const wdb_gather_field &fd, int p) {
  return fd.policy_mask == 0 || ((fd.policy_mask >> p) & 1);
}

// destination d of policy p and its row width (selects, not an indexed load: a parameter array
// indexed at run time would be staged through local memory)
__device__ __forceinline__ float *dst_rows(const FieldsArgs &a, int p, int d) {
  return d ? a.rows[p][1] : a.rows[p][0];
}
__device__ __forceinline__ int dst_pitch(const FieldsArgs &a, int p, int d) {
  return d ? a.dst_width[p][1] : a.dst_width[p][0];
}

// row part: one warp per (policy, env, slot) row; per agent-first field, lanes over its
// elements.  tile part: one CTA per tile of an agent-last field, read column by column
// (consecutive agents are consecutive in the source) and written row by row.  int32 keys and
// masks are converted to float32 on the way.
__global__ void __launch_bounds__(kGenThreads)
gather_fields_kernel(const __grid_constant__ FieldsArgs a) {
  if (blockIdx.x >= a.row_blocks) {
    __shared__ float tile[kTileElems + 32];
    const long long t = blockIdx.x - a.row_blocks;
    int j = 0;
    for (int q = 1; q < a.n_jobs; q++)
      if (t >= a.job[q].first) j = q;
    const TileJob &jb = a.job[j];
    const wdb_gather_field &fd = a.field[jb.f];
    const int p = jb.p, np = a.np[p];
    const long long per_env = (long long)jb.tiles_a * jb.tiles_c;
    const long long r = t - jb.first;
    const int env = (int)(r / per_env);
    const int rem = (int)(r - env * per_env);
    const int a0 = (rem / jb.tiles_c) * jb.ta, c0 = (rem % jb.tiles_c) * jb.tc;
    const int na = min(jb.ta, np - a0), nc = min(jb.tc, fd.width - c0);
    const int ns = fd.own_rows ? np : a.n_agents;
    const int *ids = fd.own_rows ? nullptr : a.ids[p];
    const int pitch = jb.ta + 1;
    const long long base = (long long)env * fd.width + c0;
    for (int k = threadIdx.x; k < nc * na; k += blockDim.x) {
      const int c = k / na, s = k - c * na;
      const long long off = (base + c) * ns + (ids ? ids[a0 + s] : a0 + s);
      tile[c * pitch + s] = fd.is_int32 ? (float)reinterpret_cast<const int *>(fd.src)[off]
                                        : reinterpret_cast<const float *>(fd.src)[off];
    }
    __syncthreads();
    const int w = dst_pitch(a, p, fd.dst);
    float *dst = dst_rows(a, p, fd.dst) + ((long long)env * np + a0) * w + fd.col + c0;
    for (int k = threadIdx.x; k < na * nc; k += blockDim.x) {
      const int s = k / nc, c = k - s * nc;
      dst[(long long)s * w + c] = tile[c * pitch + s];
    }
    return;
  }
  const int lane = threadIdx.x & 31;
  const long long warp = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (warp >= a.first_item[a.n_policies]) return;
  int p = 0;
#pragma unroll
  for (int q = 1; q < 4; q++)
    if (q < a.n_policies && warp >= a.first_item[q]) p = q;
  const long long r = warp - a.first_item[p];
  const int np = a.np[p];
  const int env = (int)(r / np), slot = (int)(r - (long long)env * np);
  const long long src_row = (long long)env * a.n_agents + (a.ids[p] ? a.ids[p][slot] : slot);
  for (int f = 0; f < a.n_fields; f++) {
    const wdb_gather_field &fd = a.field[f];
    float *dst = dst_rows(a, p, fd.dst);
    if (!dst || fd.agents_last || !feeds(fd, p)) continue;
    dst += r * dst_pitch(a, p, fd.dst) + fd.col;
    const long long row = fd.own_rows ? r : src_row;
    if (fd.is_int32) {
      const int *src = reinterpret_cast<const int *>(fd.src) + row * fd.width;
      for (int i = lane; i < fd.width; i += 32) dst[i] = (float)src[i];
    } else {
      const float *src = reinterpret_cast<const float *>(fd.src) + row * fd.width;
      for (int i = lane; i < fd.width; i += 32) dst[i] = src[i];
    }
  }
}

struct BookArgs {
  int n_envs, n_agents, n_policies;
  const int *done;
  int *done_batch;
  int *step_running_sum;
  unsigned long long *episodic_step_sum, *num_completed;
  int np[4];
  const int *ids[4];
  const float *rewards[4];     // the policy's own [E, Np] array, or the shared [E, N] one
  const int *actions[4];       // the same for [E, Np | N, n_heads[p]]
  int own_rewards[4], own_actions[4], n_heads[4];
  float *rewards_batch[4];
  int *actions_batch[4];
  float *reward_running_sum[4];
  float *episodic_reward_sum[4];
};

// one CTA per env
__global__ void __launch_bounds__(kGenThreads)
bookkeep_kernel(const __grid_constant__ BookArgs b) {
  const int env = blockIdx.x, tid = threadIdx.x;
  const int raw = b.done[env];
  const bool d = raw > 0;                     // any non-zero flag ends the episode
  __shared__ float red[kGenThreads / 32];
  for (int p = 0; p < b.n_policies; p++) {
    const int np = b.np[p], nh = b.n_heads[p];
    float part = 0.0f;
    for (int slot = tid; slot < np; slot += blockDim.x) {
      const int agent = b.ids[p] ? b.ids[p][slot] : slot;
      const long long shared = (long long)env * b.n_agents + agent;
      const long long dst = (long long)env * np + slot;
      const float r = b.rewards[p][b.own_rewards[p] ? dst : shared];
      if (b.rewards_batch[p]) b.rewards_batch[p][dst] = r;
      if (b.actions[p] && b.actions_batch[p]) {
        const long long src = b.own_actions[p] ? dst : shared;
        for (int k = 0; k < nh; k++)
          b.actions_batch[p][dst * nh + k] = b.actions[p][src * nh + k];
      }
      if (b.reward_running_sum[p]) {
        const float run = b.reward_running_sum[p][dst] + r;
        b.reward_running_sum[p][dst] = d ? 0.0f : run;
        if (d) part += run;
      }
    }
    if (d && b.episodic_reward_sum[p] && b.reward_running_sum[p]) {   // CTA-uniform branch
#pragma unroll
      for (int off = 16; off > 0; off >>= 1) part += __shfl_down_sync(0xffffffffu, part, off);
      if ((tid & 31) == 0) red[tid >> 5] = part;
      __syncthreads();
      if (tid == 0) {
        float s = 0.0f;
        for (int w = 0; w < (int)(blockDim.x >> 5); w++) s += red[w];
        atomicAdd(b.episodic_reward_sum[p], s);
      }
      __syncthreads();
    }
  }
  if (tid == 0) {
    if (b.done_batch) b.done_batch[env] = raw;    // the batch keeps the raw flag (MountainCar: 2)
    if (b.step_running_sum) {
      const int steps = b.step_running_sum[env] + 1;
      b.step_running_sum[env] = d ? 0 : steps;
      if (d && b.episodic_step_sum) atomicAdd(b.episodic_step_sum, (unsigned long long)steps);
    }
    if (d && b.num_completed) atomicAdd(b.num_completed, 1ull);
  }
}

}  // namespace

WDB_API int wdb_gather_policy_rows(void *stream, const wdb_gather *g) {
  if (!g || !g->full || g->n_envs < 1 || g->n_agents < 1 || g->width < 1 ||
      g->n_policies < 1 || g->n_policies > 4)
    return (int)cudaErrorInvalidValue;
  GatherArgs a = {};
  a.n_envs = g->n_envs; a.n_agents = g->n_agents; a.width = g->width;
  a.n_policies = g->n_policies; a.scatter = g->scatter ? 1 : 0;
  a.full = reinterpret_cast<uint32_t *>(g->full);
  long long items = 0;
  for (int p = 0; p < g->n_policies; p++) {
    if (!g->policy[p].rows || g->policy[p].n_agents < 1 || g->policy[p].n_agents > g->n_agents)
      return (int)cudaErrorInvalidValue;
    a.np[p] = g->policy[p].n_agents;
    a.ids[p] = g->policy[p].agent_ids;
    a.rows[p] = reinterpret_cast<uint32_t *>(g->policy[p].rows);
    a.first_item[p] = items;
    items += (long long)g->n_envs * a.np[p];
  }
  for (int p = g->n_policies; p <= 4; p++) a.first_item[p] = items;
  const long long threads = items * 32;
  gather_rows_kernel<<<(unsigned)((threads + kGenThreads - 1) / kGenThreads), kGenThreads, 0,
                       as_stream(stream)>>>(a);
  return finish_launch();
}

WDB_API int wdb_gather_policy_fields(void *stream, const wdb_gather_fields *g) {
  if (!g || g->n_envs < 1 || g->n_agents < 1 || g->n_policies < 1 || g->n_policies > 4 ||
      g->n_fields < 1 || g->n_fields > WDB_GATHER_MAX_FIELDS)
    return (int)cudaErrorInvalidValue;
  FieldsArgs a = {};
  a.n_envs = g->n_envs; a.n_agents = g->n_agents;
  a.n_policies = g->n_policies; a.n_fields = g->n_fields;
  for (int p = 0; p < g->n_policies; p++) {
    const wdb_gather_fields_policy &io = g->policy[p];
    if (io.n_agents < 1 || io.n_agents > g->n_agents) return (int)cudaErrorInvalidValue;
    a.np[p] = io.n_agents;
    a.ids[p] = io.agent_ids;
    for (int d = 0; d < 2; d++) {
      a.rows[p][d] = io.rows[d];
      a.dst_width[p][d] = io.dst_width[d] > 0 ? io.dst_width[d] : g->dst_width[d];
    }
  }
  bool has_rows[4] = {false, false, false, false};
  for (int f = 0; f < g->n_fields; f++) {
    const wdb_gather_field &fd = g->field[f];
    const unsigned mask = (unsigned)fd.policy_mask;
    if (!fd.src || fd.width < 1 || fd.dst < 0 || fd.dst > 1 || fd.col < 0 ||
        (mask >> g->n_policies) != 0u || (fd.own_rows && __builtin_popcount(mask) != 1))
      return (int)cudaErrorInvalidValue;
    a.field[f] = fd;
    // one source agent: agent-last and agent-first are the same memory, and a warp per row
    // moves it without a tile
    if (fd.agents_last) {
      int ns = g->n_agents;
      for (int p = 0; p < g->n_policies; p++)
        if (fd.own_rows && feeds(fd, p)) ns = a.np[p];
      if (ns == 1) a.field[f].agents_last = 0;
    }
    for (int p = 0; p < g->n_policies; p++) {
      if (!feeds(fd, p)) continue;
      if (fd.col + fd.width > a.dst_width[p][fd.dst]) return (int)cudaErrorInvalidValue;
      if (!a.rows[p][fd.dst]) continue;
      if (!a.field[f].agents_last) {
        has_rows[p] = true;
        continue;
      }
      if (a.n_jobs == kMaxTileJobs) return (int)cudaErrorInvalidValue;
      TileJob &jb = a.job[a.n_jobs++];
      jb.p = p; jb.f = f;
      jb.tc = fd.width < 32 ? fd.width : 32;
      const int np32 = (a.np[p] + 31) / 32 * 32;
      const int ta = kTileElems / jb.tc / 32 * 32;
      jb.ta = ta < np32 ? ta : np32;
      jb.tiles_a = (a.np[p] + jb.ta - 1) / jb.ta;
      jb.tiles_c = (fd.width + jb.tc - 1) / jb.tc;
    }
  }
  long long items = 0;
  for (int p = 0; p < g->n_policies; p++) {
    a.first_item[p] = items;
    if (has_rows[p]) items += (long long)g->n_envs * a.np[p];
  }
  for (int p = g->n_policies; p <= 4; p++) a.first_item[p] = items;
  a.row_blocks = (items * 32 + kGenThreads - 1) / kGenThreads;
  long long tiles = 0;
  for (int j = 0; j < a.n_jobs; j++) {
    a.job[j].first = tiles;
    tiles += (long long)g->n_envs * a.job[j].tiles_a * a.job[j].tiles_c;
  }
  const long long blocks = a.row_blocks + tiles;
  if (blocks == 0) return (int)cudaSuccess;
  gather_fields_kernel<<<(unsigned)blocks, kGenThreads, 0, as_stream(stream)>>>(a);
  return finish_launch();
}

WDB_API int wdb_rollout_bookkeep(void *stream, const wdb_bookkeep *k) {
  if (!k || !k->done || k->n_envs < 1 || k->n_agents < 1 ||
      k->n_policies < 1 || k->n_policies > 4 || k->n_heads < 0)
    return (int)cudaErrorInvalidValue;
  BookArgs b = {};
  b.n_envs = k->n_envs; b.n_agents = k->n_agents; b.n_policies = k->n_policies;
  b.done = k->done;
  b.done_batch = k->done_batch; b.step_running_sum = k->step_running_sum;
  b.episodic_step_sum = k->episodic_step_sum; b.num_completed = k->num_completed_episodes;
  for (int p = 0; p < k->n_policies; p++) {
    const wdb_bookkeep_policy &io = k->policy[p];
    if (io.n_agents < 1 || io.n_agents > k->n_agents || io.n_heads < 0)
      return (int)cudaErrorInvalidValue;
    b.own_rewards[p] = io.rewards != nullptr;
    b.rewards[p] = io.rewards ? io.rewards : k->rewards;
    b.own_actions[p] = io.actions != nullptr;
    b.actions[p] = io.actions ? io.actions : k->actions;
    b.n_heads[p] = io.actions ? io.n_heads : k->n_heads;
    if (!b.rewards[p]) return (int)cudaErrorInvalidValue;
    if (io.actions_batch && (!b.actions[p] || b.n_heads[p] < 1)) return (int)cudaErrorInvalidValue;
    b.np[p] = io.n_agents; b.ids[p] = io.agent_ids;
    b.rewards_batch[p] = io.rewards_batch; b.actions_batch[p] = io.actions_batch;
    b.reward_running_sum[p] = io.reward_running_sum;
    b.episodic_reward_sum[p] = io.episodic_reward_sum;
  }
  bookkeep_kernel<<<k->n_envs, kGenThreads, 0, as_stream(stream)>>>(b);
  return finish_launch();
}
