// wdb_tc_common.cuh -- parameter blocks and device helpers shared by the three TagContinuous
// kernels: wdb_tag_continuous.cu (whole env replicas packed into one CTA, N <= 320 and the
// single-CTA large-env variant), wdb_tc_small_v2.cu (the second-generation small-env kernel)
// and wdb_tc_wide.cu (one env spread over a thread-block cluster: blocks_per_env > 1,
// BASELINE config 4).  Everything here is exactness-critical: all kernels must rank, divide
// and sample with the SAME expressions (see the header of wdb_tag_continuous.cu for what
// "parity" means).
#pragma once
#include <math_constants.h>

#include <cuda_bf16.h>

#include "wdb_common.cuh"
#include "wdb_sortnet.cuh"

using namespace wdb;


namespace wdb {

constexpr int kMaxPolicies = 4;
constexpr int kListLen = 16;   // sorted candidate list kept per agent (self + K+1 <= 16)
constexpr int kHistCap = 32;   // history path: candidates one lane may collect

// Profiling aid (-DWDB_PHASE_CLOCKS): thread 0 of CTA 0 records the SM clock at the phase
// boundaries into stats[8 + i] (the stats buffer must then hold >= 32 ints).
#ifdef WDB_PHASE_CLOCKS
#define WDB_MARK(i)                                                                  \
  if (P.stats && blockIdx.x == 0 && threadIdx.x == 0) P.stats[8 + (i)] = (int)(clock64() - wdb_t0);
#else
#define WDB_MARK(i)
#endif

struct TcParams {
  int n_envs, N, epb, K, episode_length;
  int use_full_obs, runner_exits, stage_obs, scratch_in_smem, id_bits;
  int use_history, scr_warp_bytes;   // per-warp scratch: history candidate list / exact path
  int force_exact;                   // A/B switch: every agent takes the exact (reference-literal) path
  int full_ctas;                     // CTAs [0, full_ctas) carry epb envs each, the rest ONE env each
                                     // (the tail of the last wave as small CTAs); >= grid: all full
  int env_begin, env_end;            // the launch steps envs [env_begin, env_end) of the n_envs
                                     // (packed kernel only; every array is indexed by global env)
  float *loc_x, *loc_y, *speed, *direction, *acceleration;
  const int *agent_types;
  float *edge_pen;
  float edge_hit_penalty, grid_length;
  const float *acc_actions, *turn_actions;
  float max_speed;
  const float *skill;
  int *alive;
  float *obs;          // may be NULL in fused mode (observations only go to obs_next)
  const int *actions;  // step-only mode: input.  fused mode: output (may be NULL)
  float *g_nd;
  int *g_nid;
  int *nearest;
  float *rewards;
  const float *step_rewards;
  int *num_runners;
  float margin, tag_reward, tag_penalty, end_reward;
  int *done, *timestep;
  int *stats;
};

struct FusedParams {
  // sampler
  void *rng;
  const float *uniforms;            // optional test hook [E, N, 2]
  int n_policies, A0, A1;
  const int *agent_policy;          // [N] policy index of each agent
  const int *agent_slot;            // [N] index of the agent inside its policy
  int policy_size[kMaxPolicies];
  const float *probs0[kMaxPolicies];  // [E, Np, A0]
  const float *probs1[kMaxPolicies];  // [E, Np, A1]
  int *actions_out;                 // sampled_actions [E, N, 2]
  int *actions_head0, *actions_head1;  // optional [E, N, 1]
  // push-to-batch slots of this timestep (all optional)
  int *actions_batch[kMaxPolicies];     // [E, Np, 2]
  float *rewards_batch[kMaxPolicies];   // [E, Np]
  float *obs_next[kMaxPolicies];        // [E, Np, F] : post-step (post-reset) observations
  unsigned char *obs_tiles[kMaxPolicies];  // optional bf16 copy of obs_next in the A-operand tile
                                           // layout of wdb_mlp_policy_forward_tiles
  int *done_batch;                      // [E]
  // episodic bookkeeping (optional)
  float *reward_running_sum[kMaxPolicies];   // [E, Np]
  float *episodic_reward_sum[kMaxPolicies];  // scalar
  int *step_running_sum;                     // [E]
  unsigned long long *episodic_step_sum, *num_completed;
  // done-masked reset
  const wdb_reset_desc *reset_table;
  int n_reset;
  const float *obs_at_reset;        // [E, N, F] (for obs_next of envs that reset)
  int do_reset;
  int pdl;                          // host only: launch programmatically dependent on the forward
  int actions_in;                   // host only: actions_batch already holds the actions (the
                                    // packed kernel's ACTS_IN instance reads them)
};

struct V2Params {
  int chunk_rows;        // rows of the observation tile (multiple of 4)
  int tile_bytes;
};

struct WideParams {
  int C;            // CTAs per env (cluster size)
  int S;            // agents per CTA slice (id order): ceil(N / C)
  int nbins;        // x-bins (power of two <= 64); bin `nbins` holds the dead agents
  int npad;         // sorted planes length: round_up(N, 16), all +inf behind the alive agents
  int sw;           // staging row pitch in floats (odd)
  int fpp;          // feature planes per staging pass (7: one pass ... 1: seven passes)
  int o_idcol;      // byte offset of the id columns inside a warp's scratch
  int o_rowptr;     // ... of the 32 x 2 destination row pointers (the staging rows follow)
  int use_window;   // 0: scan every alive agent (A/B switch)
  // byte offsets into dynamic shared memory (identical in every CTA: DSMEM addressing)
  int o_pos, o_sp, o_acc, o_dir, o_alive, o_cross, o_type, o_kx, o_ky, o_sid, o_tag,
      o_tagcnt, o_wcount, o_binbase, o_leftmax, o_rightmin, o_misc, o_tab, o_scr, o_stage,
      o_exact;
  int scr_warp_bytes, stage_warp_bytes;
};

// One TagContinuous launch as tc_plan decided it: which kernel, and its geometry.
struct TcPlan {
  enum Kernel { kPacked, kV2, kWide } kernel;
  int grid, block;
  int cluster;      // kWide: CTAs per env, launched as one thread-block cluster
  int minb;         // kV2: CTAs per SM the kernel instance is built for (3, 4 or 7)
  size_t smem;      // dynamic shared memory per CTA
  V2Params v2;      // kV2 only
  WideParams wide;  // kWide only
};

// The plan and launch halves of the cluster kernel (wdb_tc_wide.cu) and of the
// second-generation small-env kernel (wdb_tc_small_v2.cu, wdb_set_option("tc_variant", 2)).
// `fused` is NULL for the env step alone.  A plan function fills P's derived fields and
// `plan`, or returns cudaErrorInvalidValue; it makes no CUDA call.
extern int g_pdl;                   // wdb_set_option("pdl", 0/1), wdb_mlp.cu
int tc_wide_plan(TcParams &P, const FusedParams *fused, int blocks_per_env, TcPlan &plan);
int tc_wide_launch(const TcParams &P, const FusedParams *fused, const TcPlan &plan,
                   cudaStream_t st);
int tc_wide_set_option(const char *name, int value, bool *handled);
bool tc_v2_eligible(const TcParams &P, const FusedParams *fused, bool obs_tiles);
int tc_v2_plan(TcParams &P, TcPlan &plan);
int tc_v2_launch(const TcParams &P, const FusedParams *fused, const TcPlan &plan,
                 cudaStream_t st);
int tc_v2_set_option(const char *name, int value, bool *handled);
extern int g_tc_history, g_tc_force_exact, g_tc_wide_single;

}  // namespace wdb

namespace {

// programmatic dependent launch (no-ops in a grid launched without the attribute)
__device__ __forceinline__ void griddep_wait() {
  asm volatile("griddepcontrol.wait;" ::: "memory");
}
__device__ __forceinline__ void griddep_launch_dependents() {
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
}

// tag_continuous_step_pycuda.cu:7-9
__constant__ float kTwoPi = 6.283185308;
__constant__ float kEpsilon = 1.0e-10;

// Byte offsets of the small shared-memory arrays (must agree between the kernel and
// plan_packed): everything before the per-warp scratch, rounded up to 16 bytes so that the
// scratch and the big tile behind it are valid TMA (cp.async.bulk) destinations.
__host__ __device__ inline int tc_key_stride(int N) { return (N + 15) & ~15; }
__host__ __device__ inline size_t tc_small_bytes(int epb, int N) {
  const size_t b = sizeof(float) * (7ull * epb * N + 2ull * epb * tc_key_stride(N))
                   + sizeof(int) * (4ull * N + 4ull * epb + 4) + 16 /* mbarrier + pad */;
  return (b + 15) & ~(size_t)15;
}

// ---- TMA 1-D bulk copies (cp.async.bulk) + mbarrier, raw PTX for sm_90a ----
__device__ __forceinline__ uint32_t smem_u32(const void *p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ void mbar_init(uint32_t mbar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(mbar), "r"(count) : "memory");
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t mbar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(mbar), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t mbar, uint32_t parity) {
  uint32_t ok;
  do {
    asm volatile(
        "{ .reg .pred p; mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2; "
        "selp.u32 %0, 1, 0, p; }"
        : "=r"(ok) : "r"(mbar), "r"(parity) : "memory");
  } while (!ok);
}
__device__ __forceinline__ void tma_load_1d(uint32_t dst_smem, const void *src, uint32_t bytes,
                                            uint32_t mbar) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
      ::"r"(dst_smem), "l"(src), "r"(bytes), "r"(mbar) : "memory");
}
__device__ __forceinline__ void tma_store_1d(void *dst, uint32_t src_smem, uint32_t bytes) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;"
               ::"l"(dst), "r"(src_smem), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool tma_ok(const void *g, uint32_t s, size_t bytes) {
  return ((reinterpret_cast<uintptr_t>(g) | (uintptr_t)s | bytes) & 15) == 0 && bytes > 0;
}

// ComputeDistance (:13-26) -- the reference's exact expression (float args, int exponent:
// resolves to the double pow, double sqrt, narrowed to float).
__device__ __forceinline__ float exact_distance(float x1, float y1, float x2, float y2) {
  return sqrt(pow(x1 - x2, 2) + pow(y1 - y2, 2));
}

// Exact k-nearest selection of ONE agent, executed cooperatively by the 32 lanes of a warp:
// the reference's literal algorithm (:154-199) -- candidates in id order, float64-derived
// float distances, K rounds of "for j > i: if d[j] < d[i] swap" -- restated as a scan.
// One round of that loop leaves at position i the left-most minimum of d[i..], and every
// element that was a strict new running minimum receives the previous running minimum;
// that is an exclusive prefix-min (left-biased on ties) over positions i.., which the
// warp evaluates 32 positions at a time.  Results are bit-identical to the sequential
// loop, including the order of exact ties.
__device__ __noinline__ int exact_select_warp(const float2 *pos, const int *salive, int N,
                                              int a, int K, float *d, int *ids, int lane) {
  const unsigned full = 0xffffffffu;
  const float2 pa = pos[a];
  int nv = 0;
  for (int base = 0; base < N; base += kWarp) {            // :154-176
    const int b = base + lane;
    const bool valid = (b < N) && (b != a) && (salive[b] != 0);
    const unsigned m = __ballot_sync(full, valid);
    if (valid) {
      const int at = nv + __popc(m & ((1u << lane) - 1));
      const float2 pb = pos[b];
      ids[at] = b;
      d[at] = exact_distance(pa.x, pa.y, pb.x, pb.y);
    }
    nv += __popc(m);
  }
  __syncwarp();
  const int kk = min(nv, K);
  for (int i = 0; i < kk; i++) {                           // :179-199
    float cd = d[i];
    int cid = ids[i];
    for (int base = i + 1; base < nv; base += kWarp) {
      const int j = base + lane;
      const bool valid = j < nv;
      const float vd = valid ? d[j] : CUDART_INF_F;
      const int vid = valid ? ids[j] : -1;
      float sd = vd;                                        // inclusive left-biased min-scan
      int sid = vid;
#pragma unroll
      for (int off = 1; off < kWarp; off <<= 1) {
        const float od = __shfl_up_sync(full, sd, off);
        const int oid = __shfl_up_sync(full, sid, off);
        if (lane >= off && !(sd < od)) { sd = od; sid = oid; }
      }
      float pd = __shfl_up_sync(full, sd, 1);               // exclusive prefix incl. carry
      int pid = __shfl_up_sync(full, sid, 1);
      if (lane == 0 || !(pd < cd)) { pd = cd; pid = cid; }
      if (valid && vd < pd) { d[j] = pd; ids[j] = pid; }    // a new running minimum: swap
      const float td = __shfl_sync(full, sd, kWarp - 1);
      const int tid_ = __shfl_sync(full, sid, kWarp - 1);
      if (td < cd) { cd = td; cid = tid_; }
      __syncwarp();
    }
    if (lane == 0) { d[i] = cd; ids[i] = cid; }
    __syncwarp();
  }
  return kk;
}

// ---------------------------------------------------------------- sorting networks
// (wdb_sortnet.cuh, generated): WDB_SORT16 / WDB_BITONIC_MERGE16 operate on 16 NAMED
// registers v0..v15 -- an array indexed through nested unrolled loops ended up in local
// memory (ncu: LDL/STL inside every compare-exchange), named scalars cannot.
#define WDB_REP16(M) M(0) M(1) M(2) M(3) M(4) M(5) M(6) M(7) M(8) M(9) M(10) M(11) M(12) M(13) M(14) M(15)

// q = (float)((double)d / c) bit-exactly, with inv_c = 1.0 / c: the float64 product can
// differ from the float64 quotient by a few ulp(53), which changes the float32 rounding
// only if the product sits within those few ulp of a float32 rounding boundary (the 29
// discarded mantissa bits ~ 0x10000000).  Those (probability ~2^-26) take the real divide.
// (rare paths are kept out of line: the kernel is larger than the instruction cache, every
//  inlined copy of a ~90-instruction float64 division costs the hot path fetch stalls)
__device__ __noinline__ float true_div_f64(float d, double c) { return (float)((double)d / c); }
__device__ __forceinline__ float div_by_const_f64(float d, double c, double inv_c) {
  const double prod = (double)d * inv_c;
  const uint32_t lo = (uint32_t)__double2loint(prod) & 0x1FFFFFFFu;
  if (__builtin_expect(lo - 0x0FFFFFF8u <= 0x10u, 0)) return true_div_f64(d, c);
  return (float)prod;
}

// Inclusive float32 prefix sum of one probability row (same left-to-right additions as
// core/random.cu:62-72) followed by the reference's binary search.  Rows of <= 32 actions
// are loaded into registers and sampled there (sample_cdf_regs, which the policy forward's
// sampling epilogue calls too); longer rows build their CDF in shared memory.
__device__ __noinline__ void cdf_long_row(float *row, const float *src, int A) {
  float c = src[0];
  row[0] = c;
  for (int i = 1; i < A; i++) { c = src[i] + c; row[i] = c; }
}
__device__ __forceinline__ int sample_row(float *row, const float *src, int A, float u) {
  // src: where the probabilities are (the staged shared-memory row itself, or the global row
  // of a block that could not travel by TMA); row: shared-memory row that receives the CDF
  // of a row longer than 32
  if (A <= 32) {
    float v[32];
#pragma unroll
    for (int i = 0; i < 32; i++) v[i] = i < A ? src[i] : 0.0f;
    return sample_cdf_regs(v, A, u);
  }
  cdf_long_row(row, src, A);
  return search_index(row, 1, u, A - 1);
}

// 8 consecutive features of one observation row -> one 16-byte chunk of the bf16 A-operand
// tiles read by wdb_mlp_policy_forward_tiles (canonical K-major layout of 128-row tiles:
// element (r, k) at (r / 8) * K1 * 16 + (k / 8) * 128 + (r % 8) * 16 + (k % 8) * 2 bytes;
// K padding = 0).  `grow` = row index inside the policy's [E * Np] rows.
__device__ __noinline__ void store_obs_chunk(unsigned char *tiles, long long grow, int c,
                                                int K1, const float *src, int F) {
  float v[8];
#pragma unroll
  for (int i = 0; i < 8; i++) v[i] = (8 * c + i < F) ? src[8 * c + i] : 0.0f;
  uint4 o;
  {
    const __nv_bfloat162 h0 = __floats2bfloat162_rn(v[0], v[1]), h1 = __floats2bfloat162_rn(v[2], v[3]);
    const __nv_bfloat162 h2 = __floats2bfloat162_rn(v[4], v[5]), h3 = __floats2bfloat162_rn(v[6], v[7]);
    o.x = *reinterpret_cast<const uint32_t *>(&h0); o.y = *reinterpret_cast<const uint32_t *>(&h1);
    o.z = *reinterpret_cast<const uint32_t *>(&h2); o.w = *reinterpret_cast<const uint32_t *>(&h3);
  }
  const long long t = grow >> 7;
  const int r = (int)(grow & 127);
  *reinterpret_cast<uint4 *>(tiles + t * (128ll * K1 * 2) + (r >> 3) * (K1 * 16) + c * 128 +
                             (r & 7) * 16) = o;
}

// ---- end of a fused step, shared by the packed, second-generation and cluster kernels:
// episodic bookkeeping (trainer_base.py:514-601) and the done-masked reset.  No
// synchronisation in here: the kernels order these against the rest of the step.

// done is sticky in the reference (only the reset kernel clears it)
__device__ __forceinline__ int tc_sticky_done(int done_now, int done_prev) {
  return done_now | (done_prev > 0 ? 1 : 0);
}

// Per env, by the one thread that owns it; `done_prev` / `steps_prev` are done[env] and
// step_running_sum[env] as loaded before the step.  An env that resets in this launch gets
// done / timestep cleared here (core/reset.cu:65-75).  Returns the env's done flag.
__device__ __forceinline__ int tc_book_env(const TcParams &P, const FusedParams &Q, int env,
                                           int done_now, int done_prev, int steps_prev) {
  const int d = tc_sticky_done(done_now, done_prev);
  if (Q.done_batch) Q.done_batch[env] = d;
  const bool will_reset = d && Q.do_reset;
  if (!will_reset) { if (d) P.done[env] = 1; }
  else { P.done[env] = 0; P.timestep[env] = 0; }
  if (Q.step_running_sum) {
    const int steps = steps_prev + 1;
    if (d) {
      if (Q.episodic_step_sum) atomicAdd(Q.episodic_step_sum, (unsigned long long)steps);
      if (Q.num_completed) atomicAdd(Q.num_completed, 1ull);
      Q.step_running_sum[env] = 0;
    } else {
      Q.step_running_sum[env] = steps;
    }
  }
  return d;
}

// Per agent of policy `pol` at row `pi` of its [E, Np] batch arrays, with reward `r` and its
// env's done flag `d`; `run_prev` is reward_running_sum[pol][pi] as loaded before the step.
__device__ __forceinline__ void tc_book_agent(const FusedParams &Q, int pol, long long pi,
                                              float r, float run_prev, int d) {
#pragma unroll
  for (int p = 0; p < kMaxPolicies; p++) {
    if (p == pol) {
      if (Q.rewards_batch[p]) Q.rewards_batch[p][pi] = r;
      if (Q.reward_running_sum[p]) {
        const float run = run_prev + r;
        if (d) {
          // one atomic per agent of a finished env (rare: once per episode)
          if (Q.episodic_reward_sum[p]) atomicAdd(Q.episodic_reward_sum[p], run);
          Q.reward_running_sum[p][pi] = 0.0f;
        } else {
          Q.reward_running_sum[p][pi] = run;
        }
      }
    }
  }
}

// Done-masked reset of one finished env: every registered array from its reference
// (core/reset.cu:9-75), words w0, w0 + dw, ...; then the env's obs_at_reset rows into
// obs_next (and, with TILES, into the bf16 obs tiles), rows r0, r0 + dr, ... one warp each.
template <bool TILES>
__device__ __forceinline__ void tc_reset_env(const FusedParams &Q, int env, int N, int F,
                                             int w0, int dw, int r0, int dr, int lane) {
  for (int arr = 0; arr < Q.n_reset; arr++) {
    const wdb_reset_desc d = Q.reset_table[arr];
    const long long words = d.bytes_per_env >> 2;
    uint32_t *dst = reinterpret_cast<uint32_t *>(
        reinterpret_cast<char *>(d.dst) + (long long)env * d.bytes_per_env);
    const uint32_t *src = reinterpret_cast<const uint32_t *>(
        reinterpret_cast<const char *>(d.ref) + (long long)env * d.bytes_per_env);
    for (long long i = w0; i < words; i += dw) dst[i] = src[i];
  }
  if (!Q.obs_at_reset) return;
  const float *src = Q.obs_at_reset + (long long)env * N * F;
  for (int row = r0; row < N; row += dr) {
    const int pol = Q.agent_policy[row];
    float *dst = nullptr;
#pragma unroll
    for (int p = 0; p < kMaxPolicies; p++)
      if (p == pol && Q.obs_next[p])
        dst = Q.obs_next[p] + ((long long)env * Q.policy_size[p] + Q.agent_slot[row]) * F;
    if (dst)
      for (int f = lane; f < F; f += kWarp) dst[f] = src[(long long)row * F + f];
    if (TILES) {
#pragma unroll
      for (int p = 0; p < kMaxPolicies; p++) {
        if (p == pol && Q.obs_tiles[p]) {
          const int K1 = (F + 15) & ~15;
          if (lane < K1 / 8)
            store_obs_chunk(Q.obs_tiles[p], (long long)env * Q.policy_size[p] + Q.agent_slot[row],
                            lane, K1, src + (long long)row * F, F);
        }
      }
    }
  }
}

// Squared distance with a FIXED operation order (dx * dx rounded, then fused dy * dy + .):
// the history scan, its threshold tau, the sort keys and the exact
// check must all see the same float for the same pair of agents.
__device__ __forceinline__ float sqdist(float ax, float ay, float bx, float by) {
  const float dx = __fsub_rn(ax, bx), dy = __fsub_rn(ay, by);
  return __fmaf_rn(dy, dy, __fmul_rn(dx, dx));
}

// History-path scan step for TWO candidates (bits BIT, BIT + 1 of the word `m`): the two
// squared distances (sqdist: explicitly rounded intrinsics, never contracted), then per
// candidate one compare, one OR into the candidate bit mask and one MIN that tracks the
// smallest squared distance left OUT of the mask.
template <int BIT>
__device__ __forceinline__ void scan_pair(uint32_t &m, float &mo_a, float &mo_b, uint32_t x_lo,
                                          uint32_t x_hi, uint32_t y_lo, uint32_t y_hi,
                                          float pax, float pay, float tau) {
  const float lo = sqdist(pax, pay, __uint_as_float(x_lo), __uint_as_float(y_lo));
  const float hi = sqdist(pax, pay, __uint_as_float(x_hi), __uint_as_float(y_hi));
  m |= (lo <= tau ? (1u << BIT) : 0u) | (hi <= tau ? (2u << BIT) : 0u);
  mo_a = lo <= tau ? mo_a : fminf(mo_a, lo);
  mo_b = hi <= tau ? mo_b : fminf(mo_b, hi);
}
// 16 candidates (4 x 16-byte loads per plane), bits BIT0 .. BIT0 + 15 of `m`
template <int BIT0>
__device__ __forceinline__ void scan_16(uint32_t &m, float &mo_a, float &mo_b, const uint4 *kx4,
                                        const uint4 *ky4, float pax,
                                        float pay, float tau) {
  const uint4 X0 = kx4[0], Y0 = ky4[0], X1 = kx4[1], Y1 = ky4[1];
  const uint4 X2 = kx4[2], Y2 = ky4[2], X3 = kx4[3], Y3 = ky4[3];
  scan_pair<BIT0 + 0>(m, mo_a, mo_b, X0.x, X0.y, Y0.x, Y0.y, pax, pay, tau);
  scan_pair<BIT0 + 2>(m, mo_a, mo_b, X0.z, X0.w, Y0.z, Y0.w, pax, pay, tau);
  scan_pair<BIT0 + 4>(m, mo_a, mo_b, X1.x, X1.y, Y1.x, Y1.y, pax, pay, tau);
  scan_pair<BIT0 + 6>(m, mo_a, mo_b, X1.z, X1.w, Y1.z, Y1.w, pax, pay, tau);
  scan_pair<BIT0 + 8>(m, mo_a, mo_b, X2.x, X2.y, Y2.x, Y2.y, pax, pay, tau);
  scan_pair<BIT0 + 10>(m, mo_a, mo_b, X2.z, X2.w, Y2.z, Y2.w, pax, pay, tau);
  scan_pair<BIT0 + 12>(m, mo_a, mo_b, X3.x, X3.y, Y3.x, Y3.y, pax, pay, tau);
  scan_pair<BIT0 + 14>(m, mo_a, mo_b, X3.z, X3.w, Y3.z, Y3.w, pax, pay, tau);
}

// The same scan WITHOUT the running minimum of the unmarked candidates: callers that mark with
// a threshold inflated by 2^-17 know that everything left out is farther than that threshold,
// which is all the verification needs (9 instead of 11 instructions per candidate pair).
template <int BIT>
__device__ __forceinline__ void scan_pair_nm(uint32_t &m, uint32_t x_lo, uint32_t x_hi,
                                             uint32_t y_lo, uint32_t y_hi, float pax, float pay,
                                             float tau) {
  const float lo = sqdist(pax, pay, __uint_as_float(x_lo), __uint_as_float(y_lo));
  const float hi = sqdist(pax, pay, __uint_as_float(x_hi), __uint_as_float(y_hi));
  m |= (lo <= tau ? (1u << BIT) : 0u) | (hi <= tau ? (2u << BIT) : 0u);
}
template <int BIT0>
__device__ __forceinline__ void scan_16_nm(uint32_t &m, const uint4 *kx4, const uint4 *ky4,
                                           float pax, float pay,
                                           float tau) {
  const uint4 X0 = kx4[0], Y0 = ky4[0], X1 = kx4[1], Y1 = ky4[1];
  const uint4 X2 = kx4[2], Y2 = ky4[2], X3 = kx4[3], Y3 = ky4[3];
  scan_pair_nm<BIT0 + 0>(m, X0.x, X0.y, Y0.x, Y0.y, pax, pay, tau);
  scan_pair_nm<BIT0 + 2>(m, X0.z, X0.w, Y0.z, Y0.w, pax, pay, tau);
  scan_pair_nm<BIT0 + 4>(m, X1.x, X1.y, Y1.x, Y1.y, pax, pay, tau);
  scan_pair_nm<BIT0 + 6>(m, X1.z, X1.w, Y1.z, Y1.w, pax, pay, tau);
  scan_pair_nm<BIT0 + 8>(m, X2.x, X2.y, Y2.x, Y2.y, pax, pay, tau);
  scan_pair_nm<BIT0 + 10>(m, X2.z, X2.w, Y2.z, Y2.w, pax, pay, tau);
  scan_pair_nm<BIT0 + 12>(m, X3.x, X3.y, Y3.x, Y3.y, pax, pay, tau);
  scan_pair_nm<BIT0 + 14>(m, X3.z, X3.w, Y3.z, Y3.w, pax, pay, tau);
}

// Insert one key into the ascending named-register list v0..v15, dropping the largest:
// 16 (min, max) pairs.  A handful of candidates beyond 16 cost far less this way than a second
// 16-key sort + bitonic merge -- which a warp used to run whenever ANY of its lanes overflowed.
#define WDB_INS1(V, i) { const uint32_t lo_ = min(V##i, nk_); nk_ = max(V##i, nk_); V##i = lo_; }
#define WDB_INSERT16(V, KEY)                                                        \
  { uint32_t nk_ = (KEY);                                                           \
    WDB_INS1(V, 0) WDB_INS1(V, 1) WDB_INS1(V, 2) WDB_INS1(V, 3) WDB_INS1(V, 4) WDB_INS1(V, 5)   \
    WDB_INS1(V, 6) WDB_INS1(V, 7) WDB_INS1(V, 8) WDB_INS1(V, 9) WDB_INS1(V, 10) WDB_INS1(V, 11) \
    WDB_INS1(V, 12) WDB_INS1(V, 13) WDB_INS1(V, 14) WDB_INS1(V, 15) }

// MAXT = 320: the common geometry (EPB * N <= 320 threads, two CTAs per SM, <= 96
// registers per thread); MAXT = 1024: one env of up to 1024 agents per CTA.
// Branch-free top-16 of ALL candidates (packed squared-distance | id keys), 16 at a time:
// sort16 + half-cleaner + bitonic merger on named registers (wdb_sortnet.cuh).
__device__ __noinline__ void network_top16(float2 pa, const float *kx, const float *ky, int N,
                                           uint32_t idmask, uint32_t *out) {
  uint32_t r0, r1, r2, r3, r4, r5, r6, r7, r8, r9, r10, r11, r12, r13, r14, r15;
  const uint32_t pad_key = 0x7f800000u | idmask;
#define WDB_KEY(i)                                                                  \
  uint32_t c##i = pad_key;                                                          \
  if (base + i < N) {                                                               \
    c##i = (__float_as_uint(sqdist(pa.x, pa.y, kx[base + i], ky[base + i])) & ~idmask) \
           | (uint32_t)(base + i);                                                  \
  }
#define WDB_COPY(i) r##i = c##i;
  {
    const int base = 0;
    WDB_REP16(WDB_KEY)
    WDB_SORT16(c)
    WDB_REP16(WDB_COPY)
  }
  for (int base = kListLen; base < N; base += kListLen) {
    WDB_REP16(WDB_KEY)
    WDB_SORT16(c)
    // half-cleaner: the 16 smallest of (r ascending) U (c ascending), as a bitonic
    // sequence, then the bitonic merger restores ascending order
    r0 = min(r0, c15); r1 = min(r1, c14); r2 = min(r2, c13); r3 = min(r3, c12);
    r4 = min(r4, c11); r5 = min(r5, c10); r6 = min(r6, c9); r7 = min(r7, c8);
    r8 = min(r8, c7); r9 = min(r9, c6); r10 = min(r10, c5); r11 = min(r11, c4);
    r12 = min(r12, c3); r13 = min(r13, c2); r14 = min(r14, c1); r15 = min(r15, c0);
    WDB_BITONIC_MERGE16(r)
  }
#undef WDB_KEY
#undef WDB_COPY
  out[0] = r0; out[1] = r1; out[2] = r2; out[3] = r3; out[4] = r4; out[5] = r5;
  out[6] = r6; out[7] = r7; out[8] = r8; out[9] = r9; out[10] = r10; out[11] = r11;
  out[12] = r12; out[13] = r13; out[14] = r14; out[15] = r15;
}

// x / kTwoPi (IEEE round-to-nearest) as reciprocal multiply + one residual correction.
// Verified EXHAUSTIVELY over all 2^32 float inputs against the division for
// c = 6.283185308f, r = 1.0f / c: identical bits whenever 1e-30 < |x| < 1e30 (and for 0);
// outside that range (never reached by direction differences) the true division runs.
__device__ __forceinline__ float div_by_two_pi(float x, float c, float r) {
  const float ax = fabsf(x);
  if (__builtin_expect((ax < 1e-30f && ax > 0.0f) || ax > 1e30f, 0)) return x / c;
  const float q0 = x * r;
  const float rem = __fmaf_rn(-q0, c, x);
  return __fmaf_rn(rem, r, q0);
}

// ---- per-agent phases of the step, shared by the packed, second-generation and cluster
// kernels.  Every float expression here is the one parity depends on: keep operand order,
// double promotions and the __f*_rn intrinsics as they are.

// Philox draw of both heads' uniforms (core/random.cu:51-85): one block of agent gi's stream.
// `seed` and `off` are loaded by the caller (in its phase 0); the offset is advanced here.
__device__ __forceinline__ void tc_draw_uniforms(const FusedParams &Q, int gi,
                                                 unsigned long long seed, unsigned long long off,
                                                 float &u0, float &u1) {
  RngHeader h;
  h.seed = seed; h.n_streams = 0;
  const uint4 d = rng_draw4(h, (unsigned long long)gi, off);
  rng_offsets(Q.rng)[gi] = off + 1;
  u0 = u32_to_uniform(d.x);
  u1 = u32_to_uniform(d.y);
}

// The sampled actions of agent gi (slot `slot` of policy `pol`, np agents per env) to every
// output that is set.  A NULL actions_batch[0] disables the push to the batch for every policy;
// so does to_batch = false (the actions came from the batch).
__device__ __forceinline__ void tc_push_actions(const FusedParams &Q, int gi, int env, int pol,
                                                int np, int slot, int act0, int act1,
                                                bool to_batch = true) {
  if (Q.actions_out) *reinterpret_cast<int2 *>(Q.actions_out + 2ll * gi) = make_int2(act0, act1);
  if (Q.actions_head0) Q.actions_head0[gi] = act0;
  if (Q.actions_head1) Q.actions_head1[gi] = act1;
  if (to_batch && Q.actions_batch[0]) {
#pragma unroll
    for (int p = 0; p < kMaxPolicies; p++)
      if (p == pol && Q.actions_batch[p])
        *reinterpret_cast<int2 *>(Q.actions_batch[p] + 2ll * ((long long)env * np + slot)) =
            make_int2(act0, act1);
  }
}

struct TcMove { float x, y, sp, dir, acc, ep; bool crossed; };

// :402-465 kinematics of agent gi, same float32 expression forms as the reference, and the
// state written back.  d_acc / d_turn: the acceleration / turn table entries of its actions.
__device__ __forceinline__ TcMove tc_move_agent(const TcParams &P, int gi, float x, float y,
                                                float sp, float dir, float acc, float skill,
                                                int alive, float d_acc, float d_turn) {
  const float L = P.grid_length;
  acc += d_acc;
  dir = fmod(dir + d_turn, kTwoPi) * alive;
  if (dir < 0) dir = kTwoPi + dir;
  const float cap = P.max_speed * skill;
  sp = min(cap, max(0.0, sp + acc)) * alive;
  if ((sp <= 0.0) || (sp >= cap)) acc = 0.0;
  x += sp * cos(dir);
  y += sp * sin(dir);
  const bool crossed = (x < 0) | (x > L) | (y < 0) | (y > L);
  float ep = 0.0f;
  if (crossed) {
    if (x < 0) x = 0.0; else if (x > L) x = L;
    if (y < 0) y = 0.0; else if (y > L) y = L;
    ep = P.edge_hit_penalty;
  }
  P.loc_x[gi] = x; P.loc_y[gi] = y; P.speed[gi] = sp;
  P.direction[gi] = dir; P.acceleration[gi] = acc; P.edge_pen[gi] = ep;
  return {x, y, sp, dir, acc, ep, crossed};
}

// Tagger ids in id order (agent_types is shared by all envs), built by one warp; returns
// their count.
template <typename T>
__device__ __forceinline__ int tc_build_tagger_list(const int *stype, int N, T *stag, int lane) {
  int cnt = 0;
  for (int base = 0; base < N; base += kWarp) {
    const int j = base + lane;
    const bool is_t = (j < N) && (stype[j] == 1);
    const unsigned m = __ballot_sync(0xffffffffu, is_t);
    if (is_t) stag[cnt + __popc(m & ((1u << lane) - 1))] = (T)j;
    cnt += __popc(m);
  }
  return cnt;
}

// :296-338 the tagger that tags the runner at `pa`: the nearest of the `ntag` taggers
// stag[] within the margin, or -1.  A float32 pre-test with a guard band; only candidates
// near the margin need the reference's float64 expression.
template <typename T>
__device__ __forceinline__ int tc_tagging_tagger(const TcParams &P, float2 pa, const float2 *pos,
                                                 const T *stag, int ntag) {
  float min_dist = P.grid_length * sqrt(2.0);
  int nearest_tagger = -1;
  float min_s = CUDART_INF_F;
  for (int q = 0; q < ntag; q++) {
    const float2 pb = pos[stag[q]];
    const float dx = pa.x - pb.x, dy = pa.y - pb.y;
    min_s = fminf(min_s, dx * dx + dy * dy);
  }
  const float guard = P.margin * 1.001f;
  if (min_s > guard * guard) return -1;
  // a tagger outside the guard band is farther than the margin, so it can only be the arg-min
  // when nobody is within the margin -- and then the arg-min is not used
  for (int q = 0; q < ntag; q++) {
    const int b = stag[q];
    const float2 pb = pos[b];
    const float dx = pa.x - pb.x, dy = pa.y - pb.y;
    if (dx * dx + dy * dy > guard * guard) continue;
    const float dist = exact_distance(pa.x, pa.y, pb.x, pb.y);
    if (dist < min_dist) { min_dist = dist; nearest_tagger = b; }
  }
  return min_dist < P.margin ? nearest_tagger : -1;
}

}  // namespace
