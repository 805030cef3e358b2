// wdb_tc_wide.cu -- TagContinuous env.step() / fused rollout step for LARGE env replicas:
// one env spread over `blocks_per_env` CTAs launched as ONE THREAD-BLOCK CLUSTER
// (BASELINE config 4: 2000 envs x 1024 agents).
//
// Replaces, for blocks_per_env > 1, the reference's multi-block mode of
// CudaTagContinuousStep (example_envs/tag_continuous/tag_continuous_step_pycuda.cu:351-520)
// with its index mapping (warp_drive/cuda_includes/core/env_dim_mapper.h:22-31: agent =
// threadIdx + (blockIdx % bpe) * blockDim, env = blockIdx / bpe) and its env-wide barrier
// (core/env_thread_sync.cu:31-62: the blocks of an env spin on a byte array in global
// memory, which dead-locks unless all of them happen to be co-resident -- the reference's
// own architecture_validate.py:53-99 warns about exactly that).  Here the blocks of an env
// ARE a cluster: co-scheduled by the hardware, synchronised by barrier.cluster, exchanging
// agent state through distributed shared memory (st.shared::cluster), never through global
// memory.
//
// Design
//   phase 0  thread = agent id (unit-stride state loads, as the reference): sampling (fused
//            mode), kinematics, state written back once; every CTA PUSHES its slice of
//            (x, y, speed, acc, dir, alive, crossed) into the shared memory of all peer CTAs
//            (DSMEM), so after one cluster barrier each CTA holds the whole env on chip.
//   phase 1  every CTA builds the same x-BINNED order of the alive agents (stable counting
//            sort by floor(x * bins / L); dead agents last): sorted key planes x[], y[] and
//            the position -> agent-id map.
//   phase 2  thread = sorted position (warps are dealt round-robin over the cluster's CTAs,
//            so alive agents are balanced and warps holding only dead agents idle).
//            k-nearest selection = the temporal-coherence threshold scan of the small-env
//            kernel, but ONLY over the x-window of bins that can hold anything within the
//            threshold radius: lanes of a warp are x-neighbours, so the window is warp-
//            uniform and every shared-memory load is a broadcast.  Everything left of /
//            right of the window is bounded below by (x_self - max x on the left)^2 resp.
//            (min x on the right - x_self)^2, which enters the same "provably the reference's
//            result or fall back to the reference's literal algorithm" verification as in
//            wdb_tag_continuous.cu.  With 1024 agents and K = 10 the window holds ~15-20 % of
//            the env: the O(N^2) pair sweep of config 4 becomes ~N * 200.
//   phase 3  features, staged per warp in shared memory in two column passes (f0-f3, then
//            f4-f6 + time) and written with unit-stride row stores.
//   phase 4  rewards / tags: tag credits are INTEGER counts per tagger in each CTA's shared
//            memory, summed over the cluster through DSMEM loads after the second cluster
//            barrier (float adds of the identical tag reward, in count order: the same bits
//            as the small-env kernel's atomics); runner exits likewise.
//   phase 5  (fused mode) push rewards / done / episodic sums, done-masked reset split over
//            the cluster's threads.
//
// Parity: same expressions, same verification, same exact path (wdb_tc_common.cuh) as the
// small-env kernel; tests/test_gpu_wide.py compares against the reference's own kernel
// compiled with wkBlocksPerEnv = 2 and 4 (512 / 256 threads per block), bit for bit.
#include "wdb_tc_common.cuh"

namespace {

constexpr int kWideMaxThreads = 1024;   // one CTA may carry a whole 1024-agent env (bpe = 1)
constexpr int kWideMaxBins = 64;
constexpr int kWideCap = 32;     // candidates one lane may collect (kHistCap)

// misc words
enum { M_T = 0, M_NRUN, M_DONEPREV, M_NALIVE, M_NTAG, M_EXITS, M_LOCK, M_STEPS, M_COUNT };

// ---- cluster / DSMEM primitives (raw PTX, sm_90+) ----
__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ void cluster_arrive() {
  asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
}
__device__ __forceinline__ void cluster_wait() {
  asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}
__device__ __forceinline__ void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;\n\t"
               "barrier.cluster.wait.acquire.aligned;" ::: "memory");
}
__device__ __forceinline__ uint32_t map_to_rank(uint32_t smem_addr, uint32_t rank) {
  uint32_t r;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(smem_addr), "r"(rank));
  return r;
}
__device__ __forceinline__ void st_cluster_b32(uint32_t addr, uint32_t v) {
  asm volatile("st.shared::cluster.b32 [%0], %1;" ::"r"(addr), "r"(v) : "memory");
}
__device__ __forceinline__ void st_cluster_v2(uint32_t addr, float x, float y) {
  asm volatile("st.shared::cluster.v2.f32 [%0], {%1, %2};" ::"r"(addr), "f"(x), "f"(y) : "memory");
}
__device__ __forceinline__ void st_cluster_u8(uint32_t addr, uint32_t v) {
  asm volatile("st.shared::cluster.u8 [%0], %1;" ::"r"(addr), "r"(v) : "memory");
}
__device__ __forceinline__ int ld_cluster_s32(uint32_t addr) {
  int v;
  asm volatile("ld.shared::cluster.s32 %0, [%1];" : "=r"(v) : "r"(addr) : "memory");
  return v;
}

__device__ __forceinline__ int wide_bin(float x, float scale, int nbins) {
  // monotone non-decreasing in x (float multiply by a positive constant, truncation, clamp):
  // that is all the window bounds rely on
  const int b = (int)(x * scale);
  return b < 0 ? 0 : (b >= nbins ? nbins - 1 : b);
}

// CDF + reference binary search on a lane-strided shared-memory row (element i of this lane
// at row[i * kWarp]): conflict-free, and no per-thread 21-float row needed
__device__ __forceinline__ int sample_row_strided(float *row, const float *src, int A, float u) {
  float c = src[0];
  row[0] = c;
  for (int i = 1; i < A; i++) {      // same left-to-right float32 additions as random.cu:62-72
    c = src[i] + c;
    row[i * kWarp] = c;
  }
  return search_index(row, kWarp, u, A - 1);
}

template <bool FUSED>
__global__ void __launch_bounds__(kWideMaxThreads, 1)
tc_wide_kernel(const __grid_constant__ TcParams P, const __grid_constant__ FusedParams Q,
               const __grid_constant__ WideParams W) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int N = P.N, K = P.K, C = W.C, S = W.S;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int nw = blockDim.x >> 5;
  const int rank = (int)cluster_ctarank();
  const int env = blockIdx.x / C;
  const float L = P.grid_length;
  const unsigned full = 0xffffffffu;

  float2 *pos = reinterpret_cast<float2 *>(smem_raw + W.o_pos);      // [N] id order
  float *ssp = reinterpret_cast<float *>(smem_raw + W.o_sp);
  float *sacc = reinterpret_cast<float *>(smem_raw + W.o_acc);
  float *sdir = reinterpret_cast<float *>(smem_raw + W.o_dir);
  int *salive = reinterpret_cast<int *>(smem_raw + W.o_alive);       // before this step's tags
  unsigned char *scross = smem_raw + W.o_cross;                      // edge crossed this step
  int *stype = reinterpret_cast<int *>(smem_raw + W.o_type);
  float *skx = reinterpret_cast<float *>(smem_raw + W.o_kx);         // [npad] x-binned order
  float *sky = reinterpret_cast<float *>(smem_raw + W.o_ky);
  uint16_t *sid = reinterpret_cast<uint16_t *>(smem_raw + W.o_sid);  // position -> agent id
  uint16_t *stag = reinterpret_cast<uint16_t *>(smem_raw + W.o_tag); // tagger ids, id order
  int *tagcnt = reinterpret_cast<int *>(smem_raw + W.o_tagcnt);      // [N] credits by MY runners
  uint16_t *wcount = reinterpret_cast<uint16_t *>(smem_raw + W.o_wcount);
  int *binbase = reinterpret_cast<int *>(smem_raw + W.o_binbase);    // [nbins + 2]
  float *leftmax = reinterpret_cast<float *>(smem_raw + W.o_leftmax);    // [nbins + 1]
  float *rightmin = reinterpret_cast<float *>(smem_raw + W.o_rightmin);  // [nbins + 1]
  int *misc = reinterpret_cast<int *>(smem_raw + W.o_misc);
  float *s_tab = reinterpret_cast<float *>(smem_raw + W.o_tab);
  // per-warp scratch: [id columns | staging rows]; the candidate list of the threshold scan
  // overlays both from the start (it is dead before either is written)
  unsigned char *s_scr = smem_raw + W.o_scr + (size_t)warp * W.scr_warp_bytes;
  float *stage = reinterpret_cast<float *>(s_scr + W.stage_warp_bytes);
  float *ex_d = reinterpret_cast<float *>(smem_raw + W.o_exact);
  int *ex_ids = reinterpret_cast<int *>(ex_d + N);

  // every CTA of the cluster must have started before anybody touches its shared memory:
  // arrive now, wait right before the DSMEM push
  cluster_arrive();

  const int F = P.use_full_obs ? 7 * (N - 1) + 1 : 7 * K + 1;
  const int nbins = W.nbins, NB1 = nbins + 1;
  const int n_chunks = (N + kWarp - 1) / kWarp;        // 32-agent chunks of the env (id order)

  // ------------------------------------------------------------------ phase 0 (id order)
  const int a = rank * S + tid;
  const bool own = (tid < S) && (a < N);
  const int gi = env * N + a;
  if (tid == 0) {
    misc[M_T] = P.timestep[env] + 1;                   // :391-393 (written back at the end:
    misc[M_NRUN] = P.num_runners[env];                 //  peers read the old value meanwhile)
    misc[M_DONEPREV] = FUSED ? P.done[env] : 0;
    misc[M_EXITS] = 0;
    misc[M_LOCK] = 0;
    misc[M_STEPS] = (FUSED && Q.step_running_sum) ? Q.step_running_sum[env] : 0;
  }
  for (int i = tid; i < N; i += blockDim.x) stype[i] = P.agent_types[i];
  const int n_tab = FUSED ? Q.A0 + Q.A1 : 0;
  if (FUSED)
    for (int i = tid; i < n_tab; i += blockDim.x)
      s_tab[i] = i < Q.A0 ? P.acc_actions[i] : P.turn_actions[i - Q.A0];

  float st_x = 0.f, st_y = 0.f, st_sp = 0.f, st_dir = 0.f, st_acc = 0.f, st_skill = 0.f;
  int st_alive = 0;
  int act0 = 0, act1 = 0;
  int my_pol = 0, my_slot = 0;
  if (own) {
    st_x = P.loc_x[gi]; st_y = P.loc_y[gi]; st_sp = P.speed[gi];
    st_dir = P.direction[gi]; st_acc = P.acceleration[gi];
    st_alive = P.alive[gi];
    st_skill = P.skill[a];
    if (FUSED) { my_pol = Q.agent_policy[a]; my_slot = Q.agent_slot[a]; }
    else {
      const int2 act = *reinterpret_cast<const int2 *>(P.actions + 2ll * gi);
      act0 = act.x; act1 = act.y;
    }
  }
  if (FUSED) {
    // programmatic dependent launch: the state loads above overlapped the forward's tail, the
    // probabilities are read from here on (a no-op without the launch attribute)
    griddep_wait();
    griddep_launch_dependents();
    // categorical sampling of both heads (core/random.cu:51-85); one Philox block per agent,
    // the stream of the agent id: identical draws to the small-env kernel and the sampler
    float u0 = 0.f, u1 = 0.f;
    if (own) {
      if (Q.uniforms) {
        u0 = Q.uniforms[2ll * gi];
        u1 = Q.uniforms[2ll * gi + 1];
      } else {
        tc_draw_uniforms(Q, gi, reinterpret_cast<const RngHeader *>(Q.rng)->seed,
                         rng_offsets(Q.rng)[gi], u0, u1);
      }
      int np = 0;
      const float *g0 = nullptr, *g1 = nullptr;
#pragma unroll
      for (int p = 0; p < kMaxPolicies; p++) {
        if (p == my_pol) {
          np = Q.policy_size[p];
          const long long grow = (long long)env * np + my_slot;
          g0 = Q.probs0[p] + grow * Q.A0;
          g1 = Q.probs1[p] + grow * Q.A1;
        }
      }
      // lane-strided CDF row in the warp's scratch (ids / row pointers / staging rows all
      // come later; the host sizes the scratch for A x 32 floats)
      float *row = reinterpret_cast<float *>(s_scr) + lane;
      act0 = sample_row_strided(row, g0, Q.A0, u0);
      act1 = sample_row_strided(row, g1, Q.A1, u1);
      tc_push_actions(Q, gi, env, my_pol, np, my_slot, act0, act1);
    }
    __syncthreads();   // s_tab staged
  }

  cluster_wait();     // all peers are running: their shared memory may be written
  if (own) {
    const int alive = st_alive;
    const TcMove mv = tc_move_agent(P, gi, st_x, st_y, st_sp, st_dir, st_acc, st_skill, alive,
                                    FUSED ? s_tab[act0] : P.acc_actions[act0],
                                    FUSED ? s_tab[Q.A0 + act1] : P.turn_actions[act1]);
    const float x = mv.x, y = mv.y, sp = mv.sp, dir = mv.dir, acc = mv.acc;
    const bool crossed = mv.crossed;
    // the whole env on chip in EVERY CTA of the cluster: local store + DSMEM push to the peers
    pos[a] = make_float2(x, y);
    ssp[a] = sp; sacc[a] = acc; sdir[a] = dir;
    salive[a] = alive;
    scross[a] = crossed ? 1 : 0;
    const uint32_t b_pos = smem_u32(&pos[a]), b_sp = smem_u32(&ssp[a]), b_acc = smem_u32(&sacc[a]),
                   b_dir = smem_u32(&sdir[a]), b_al = smem_u32(&salive[a]),
                   b_cr = smem_u32(&scross[a]);
    for (int r = 1; r < C; r++) {
      const uint32_t peer = (uint32_t)((rank + r) % C);
      st_cluster_v2(map_to_rank(b_pos, peer), x, y);
      st_cluster_b32(map_to_rank(b_sp, peer), __float_as_uint(sp));
      st_cluster_b32(map_to_rank(b_acc, peer), __float_as_uint(acc));
      st_cluster_b32(map_to_rank(b_dir, peer), __float_as_uint(dir));
      st_cluster_b32(map_to_rank(b_al, peer), (uint32_t)alive);
      st_cluster_u8(map_to_rank(b_cr, peer), crossed ? 1u : 0u);
    }
  }
  cluster_sync_all();   // #1: every CTA holds the post-kinematics state of the whole env

  const int t_env = misc[M_T];
  const int g_nrun = misc[M_NRUN];
  const int done_prev = misc[M_DONEPREV];

  // tagger id list, built by warp 0
  if (warp == 0) {
    const int cnt = tc_build_tagger_list(stype, N, stag, lane);
    if (lane == 0) misc[M_NTAG] = cnt;
  }

  // ------------------------------------------------------------------ phase 1: x-binned order
  // Stable counting sort of the agents by (alive ? x-bin : nbins): deterministic (order inside
  // a bin = id order), computed redundantly by every CTA from its own copy of the env.
  const float binscale = (float)nbins / L;
  uint32_t *binmax_u = reinterpret_cast<uint32_t *>(leftmax);    // per-bin max / min x first,
  uint32_t *binmin_u = reinterpret_cast<uint32_t *>(rightmin);   // prefix / suffix in place later
  if (!P.use_full_obs) {
    for (int i = tid; i < n_chunks * NB1; i += blockDim.x) wcount[i] = 0;
    for (int i = tid; i < NB1; i += blockDim.x) { binmax_u[i] = 0u; binmin_u[i] = 0x7f800000u; }
    for (int i = tid; i < W.npad; i += blockDim.x) { skx[i] = CUDART_INF_F; sky[i] = CUDART_INF_F; }
    __syncthreads();
    for (int cw = warp; cw < n_chunks; cw += nw) {
      const int j = cw * kWarp + lane;
      int b = NB1;                                       // lanes beyond N: their own group
      if (j < N) {
        const float x = pos[j].x;
        b = salive[j] ? wide_bin(x, binscale, nbins) : nbins;
        if (salive[j]) {                                 // x >= 0: uint order == float order
          atomicMax(&binmax_u[b], __float_as_uint(x));
          atomicMin(&binmin_u[b], __float_as_uint(x));
        }
      }
      const unsigned m = __match_any_sync(full, b);
      if (j < N && (m & ((1u << lane) - 1)) == 0) wcount[cw * NB1 + b] = (uint16_t)__popc(m);
    }
    __syncthreads();
    // per bin: exclusive prefix over the chunks; then the exclusive prefix over the bins
    for (int b = tid; b < NB1; b += blockDim.x) {
      int run = 0;
      for (int cw = 0; cw < n_chunks; cw++) {
        const int t = wcount[cw * NB1 + b];
        wcount[cw * NB1 + b] = (uint16_t)run;
        run += t;
      }
      binbase[b + 1] = run;      // bin totals, scanned below
    }
    __syncthreads();
    if (tid == 0) {
      int run = 0;
      float lm = -CUDART_INF_F;
      for (int b = 0; b < NB1; b++) {
        const int t = binbase[b + 1];
        const float bm = (b < nbins && t > 0) ? __uint_as_float(binmax_u[b]) : -CUDART_INF_F;
        binbase[b] = run;
        run += t;
        leftmax[b] = lm;          // max x over the alive agents in bins < b
        lm = fmaxf(lm, bm);
      }
      binbase[NB1] = run;
      misc[M_NALIVE] = binbase[nbins];
      float rm = CUDART_INF_F;
      for (int b = nbins - 1; b >= 0; b--) {
        const bool any = binbase[b + 1] > binbase[b];
        const float bm = any ? __uint_as_float(binmin_u[b]) : CUDART_INF_F;
        rightmin[b] = rm;         // min x over the alive agents in bins > b
        rm = fminf(rm, bm);
      }
    }
    __syncthreads();
    for (int cw = warp; cw < n_chunks; cw += nw) {
      const int j = cw * kWarp + lane;
      int b = NB1;
      if (j < N) b = salive[j] ? wide_bin(pos[j].x, binscale, nbins) : nbins;
      const unsigned m = __match_any_sync(full, b);
      if (j < N) {
        const int q = binbase[b] + wcount[cw * NB1 + b] + __popc(m & ((1u << lane) - 1));
        sid[q] = (uint16_t)j;
        if (salive[j]) { skx[q] = pos[j].x; sky[q] = pos[j].y; }
      }
    }
    __syncthreads();
  } else {
    __syncthreads();
  }
  // tag credit counters (they overlay the counting-sort table, dead from here on)
  for (int i = tid; i < N; i += blockDim.x) tagcnt[i] = 0;
  __syncthreads();
  const int n_alive = P.use_full_obs ? 0 : misc[M_NALIVE];

  // ------------------------------------------------------------------ phases 2-4 (sorted order)
  // warps are dealt round-robin over the CTAs of the cluster: alive agents sit first in the
  // order, so every CTA gets its share and warps past the alive count have nothing to search
  const int q = (warp * C + rank) * kWarp + lane;
  const bool have = q < N;
  int a2 = 0;
  bool alive = false;
  if (!P.use_full_obs) {
    a2 = have ? (int)sid[q] : 0;
    alive = have && (q < n_alive);
  } else {
    a2 = have ? q : 0;                     // full observation: no search, identity order
    alive = have && salive[a2] != 0;
  }
  const int gi2 = env * N + a2;

  const double diag = sqrt(2.0) * L;                // :94
  const double inv_diag = 1.0 / diag;
  const float vnorm = P.max_speed + kEpsilon;       // :101
  const float two_pi = kTwoPi, inv_two_pi = 1.0f / kTwoPi;

  if (!P.use_full_obs) {
    uint32_t R[kListLen];
    int kk = 0;
    bool suspect = false;
    int idbits = 1;
    while ((1 << idbits) < W.npad) idbits++;
    const uint32_t idmask = (1u << idbits) - 1u;
    const bool net_ok = (K + 2 <= kListLen);
    const float2 pa = pos[a2];
    uint16_t *lst = reinterpret_cast<uint16_t *>(s_scr) + lane;     // candidate positions column
    const int nv = n_alive - 1;                                      // alive others
    if (alive) kk = min(nv, K);
    // ---- threshold from last step's neighbours (any value is safe, see the verification)
    float tau = -1.0f;
    if (alive && net_ok && P.use_history) {
      int seen = 0;
      float t = 0.0f;
      const int *nn = P.nearest + (long long)gi2 * K;
      for (int p = 0; p < K; p++) {
        const int b = min(max(nn[p], 0), N - 1);
        if (b != a2 && salive[b]) {
          const float2 pb = pos[b];
          t = fmaxf(t, sqdist(pa.x, pa.y, pb.x, pb.y));
          seen++;
        }
      }
      if (seen < kk) t *= 1.0f + 0.9f * (float)(kk - seen);
      if (seen > 0) tau = t;
    }
    // ---- threshold scan over a warp-uniform x-window of bins, at most two passes: a lane
    // whose candidate list came out too long (> kWideCap) or too short (< kk + 1) retries once
    // with a smaller / larger disc before the branch-free network has to run.  ANY threshold is
    // safe: the verification below only uses "everything not in the list is farther than
    // m_out".
    int cnt = 0;
    float m_out = CUDART_INF_F;
    bool hist = false;
    // first-pass overflow whose retry failed: the K nearest still lie inside the FIRST window,
    // so the network runs over that window only
    bool overflow = false;
    int win_lo = 0, win_n = 0, cnt0 = 0;
    float m_edge0 = CUDART_INF_F;
    {
      bool want = alive && net_ok && tau >= 0.0f;
      bool over0 = false;
#pragma unroll 1
      for (int pass = 0; pass < 2; pass++) {
        int blo = 0x7fffffff, bhi = -1;
        if (want) {
          const float rad = sqrtf(tau) * 1.000001f + 1e-30f;
          blo = wide_bin(fmaxf(pa.x - rad, 0.0f), binscale, nbins);
          bhi = wide_bin(fminf(pa.x + rad, L), binscale, nbins);
        }
        int wlo = __reduce_min_sync(full, blo), whi = __reduce_max_sync(full, bhi);
        if (whi < 0) break;                      // no lane scans (warp-uniform)
        if (!W.use_window) { wlo = 0; whi = nbins - 1; }
        const int lo16 = binbase[wlo] & ~15;
        const int hi16 = min((binbase[whi + 1] + 15) & ~15, W.npad);
        float mo_a = CUDART_INF_F, mo_b = CUDART_INF_F;
        const float tau_s = want ? tau : -1.0f;          // the other lanes mark nothing
        int c = 0;
        for (int j = lo16; j < hi16; j += 32) {
          uint32_t m = 0;
          const uint4 *kx4 = reinterpret_cast<const uint4 *>(skx + j);
          const uint4 *ky4 = reinterpret_cast<const uint4 *>(sky + j);
          scan_16<0>(m, mo_a, mo_b, kx4, ky4, pa.x, pa.y, tau_s);
          if (j + 16 < hi16) scan_16<16>(m, mo_a, mo_b, kx4 + 4, ky4 + 4, pa.x, pa.y, tau_s);
          for (; m; m &= m - 1) {
            if (c < kWideCap) lst[c * kWarp] = (uint16_t)(j + __ffs(m) - 1);
            c++;
          }
        }
        bool good = false;
        if (want) {
          // everything outside the window: bins < wlo lie at or left of leftmax[wlo], bins >
          // whi at or right of rightmin[whi] (empty side: -inf / +inf -> bound +inf).
          // dx = fl(x_self - x_other) is monotone in x_other, fl(dx * dx) in |dx|, and the
          // fused dy * dy + . only adds: a rigorous lower bound of sqdist() for all of them
          const float dl = pa.x - leftmax[wlo], dr = rightmin[whi] - pa.x;
          const float m_edge = fminf(__fmul_rn(dl, dl), __fmul_rn(dr, dr));
          m_out = fminf(fminf(mo_a, mo_b), m_edge);
          cnt = c;
          good = (c >= kk + 1) && (c <= kWideCap);
          if (pass == 0) { over0 = c > kWideCap; cnt0 = c; m_edge0 = m_edge; }
        }
        if (pass == 0) { win_lo = lo16; win_n = hi16 - lo16; }
        hist = hist || good;
        want = want && !good && pass == 0;
        if (want) tau = (c > kWideCap) ? tau * (20.0f / (float)c) : tau * 2.5f;
      }
      overflow = over0 && !hist;
    }
    if (alive && net_ok) {
      uint32_t r0, r1, r2, r3, r4, r5, r6, r7, r8, r9, r10, r11, r12, r13, r14, r15;
      int n_have = min(nv, kListLen - 1);
      int n_cand = nv;
      if (hist) {
#define WDB_HKEY(i)                                                                 \
  uint32_t c##i;                                                                    \
  {                                                                                 \
    const int b = min((int)lst[(hbase + i) * kWarp], W.npad - 1);                   \
    const uint32_t key = (__float_as_uint(sqdist(pa.x, pa.y, skx[b], sky[b])) & ~31u) \
                         | (uint32_t)(hbase + i);                                   \
    c##i = (hbase + i < cnt) ? key : (0x7f800000u | 31u);                           \
  }
#pragma unroll 1
        for (int hbase = 0; hbase < kWideCap; hbase += kListLen) {
          if (hbase >= cnt) break;
          WDB_REP16(WDB_HKEY)
          WDB_SORT16(c)
          if (hbase == 0) {
            r0 = c0; r1 = c1; r2 = c2; r3 = c3; r4 = c4; r5 = c5; r6 = c6; r7 = c7;
            r8 = c8; r9 = c9; r10 = c10; r11 = c11; r12 = c12; r13 = c13; r14 = c14;
            r15 = c15;
          } else {
            r0 = min(r0, c15); r1 = min(r1, c14); r2 = min(r2, c13); r3 = min(r3, c12);
            r4 = min(r4, c11); r5 = min(r5, c10); r6 = min(r6, c9); r7 = min(r7, c8);
            r8 = min(r8, c7); r9 = min(r9, c6); r10 = min(r10, c5); r11 = min(r11, c4);
            r12 = min(r12, c3); r13 = min(r13, c2); r14 = min(r14, c1); r15 = min(r15, c0);
            WDB_BITONIC_MERGE16(r)
          }
        }
#undef WDB_HKEY
        n_have = min(cnt - 1, kListLen - 1);
        n_cand = cnt - 1;
      } else {
        // no usable threshold (first step after a reset, list under/overflow): branch-free
        // top-16 of all alive agents (they are the first n_alive positions of the planes)
        if (P.stats && P.use_history) atomicAdd(&P.stats[overflow ? 3 : 2], 1);
        uint32_t out[kListLen];
        if (overflow) {
          // every agent within tau (> kWideCap of them, the K nearest included) sits in the
          // window [win_lo, win_lo + win_n); everything outside is bounded below by m_edge
          network_top16(pa, skx + win_lo, sky + win_lo, win_n, idmask, out);
          m_out = m_edge0;
          n_cand = cnt0 - 1;
        } else {
          m_out = CUDART_INF_F;
          win_lo = 0;
          network_top16(pa, skx, sky, (n_alive + 15) & ~15, idmask, out);
        }
        r0 = out[0]; r1 = out[1]; r2 = out[2]; r3 = out[3]; r4 = out[4]; r5 = out[5];
        r6 = out[6]; r7 = out[7]; r8 = out[8]; r9 = out[9]; r10 = out[10]; r11 = out[11];
        r12 = out[12]; r13 = out[13]; r14 = out[14]; r15 = out[15];
      }
      R[0] = r0; R[1] = r1; R[2] = r2; R[3] = r3; R[4] = r4; R[5] = r5; R[6] = r6;
      R[7] = r7; R[8] = r8; R[9] = r9; R[10] = r10; R[11] = r11; R[12] = r12;
      R[13] = r13; R[14] = r14; R[15] = r15;
      // The id field of a key is the index into the candidate list on the threshold path (5
      // bits: the squared distance keeps 18 mantissa bits) and the sorted position on the
      // network path (up to 10-11 bits).  floor_out = the truncated distance of winner K+1
      // bounds everything ranked behind it; then the keys are replaced by positions.
      const uint32_t idm = hist ? 31u : idmask;
      uint32_t last_key = 0;
#pragma unroll
      for (int i = 1; i < kListLen; i++) last_key = (i == K + 1) ? R[i] : last_key;
      const float floor_out = __uint_as_float(last_key & ~idm);
#pragma unroll
      for (int i = 0; i < kListLen; i++)
        R[i] = hist ? (uint32_t)min((int)lst[(R[i] & 31u) * kWarp], W.npad - 1)
                    : (R[i] & idmask) + (uint32_t)win_lo;
      // ---- verification on EXACT float32 squared distances of the K+1 nearest (same rules
      // as wdb_tag_continuous.cu: strictly increasing with relative gaps > 2^-19, and
      // everything not examined clears the K-th by the same margin)
      const int m = min(n_have, K + 1);
      if ((int)R[0] != q) suspect = true;     // a co-located agent sorted first
      float es[kListLen];
      bool misordered = false;
      {
        float prev = 0.0f;
#pragma unroll
        for (int i = 1; i < kListLen; i++) {
          es[i] = CUDART_INF_F;
          if (i <= m) {
            const int c = min((int)R[i], W.npad - 1);
            es[i] = sqdist(pa.x, pa.y, skx[c], sky[c]);
            misordered |= !(es[i] > prev);
            prev = es[i];
          }
        }
      }
      if (misordered) {
#pragma unroll 1
        for (int pass = 0; pass < kListLen - 1; pass++) {
#pragma unroll
          for (int i = 1; i + 1 < kListLen; i++) {
            if (((i + pass) & 1) == 0) continue;
            const bool sw = es[i + 1] < es[i];
            const float ts = es[i]; const uint32_t tr = R[i];
            es[i] = sw ? es[i + 1] : ts;   R[i] = sw ? R[i + 1] : tr;
            es[i + 1] = sw ? ts : es[i + 1]; R[i + 1] = sw ? tr : R[i + 1];
          }
        }
      }
      {
        float prev = 0.0f;
#pragma unroll
        for (int i = 1; i < kListLen; i++) {
          if (i <= m) {
            if (!(es[i] - prev > es[i] * 1.9073486328125e-06f)) suspect = true;
            prev = es[i];
          }
        }
        float rest = m_out;
        if (n_cand > K + 1) rest = fminf(rest, floor_out);
        if (rest < CUDART_INF_F && m >= K) {
          float xk = 0.0f;
#pragma unroll
          for (int i = 1; i < kListLen; i++) xk = (i == K) ? es[i] : xk;
          if (!(rest - xk > rest * 1.9073486328125e-06f)) suspect = true;
        }
      }
      // positions -> agent ids
#pragma unroll
      for (int i = 1; i < kListLen; i++)
        if (i <= kk) R[i] = (uint32_t)sid[min((int)R[i], N - 1)];
    } else if (alive) {
      suspect = true;
    }
    if (P.force_exact && alive) suspect = true;
    // ---- exact path: the reference's literal algorithm, one suspect agent at a time per
    // warp, on the CTA's one scratch list pair (rare: a spin lock serialises the warps)
    unsigned todo = __ballot_sync(full, suspect);
    uint16_t *idcol = reinterpret_cast<uint16_t *>(s_scr + W.o_idcol) + lane;
    if (todo) {
      if (lane == 0) {
        while (atomicCAS(&misc[M_LOCK], 0, 1) != 0) __nanosleep(64);
      }
      __syncwarp();
      while (todo) {
        const int Lx = __ffs(todo) - 1;
        todo &= todo - 1;
        const int ax = __shfl_sync(full, a2, Lx);
        const int kx = exact_select_warp(pos, salive, N, ax, K, ex_d, ex_ids, lane);
        if (lane == Lx) {
          kk = kx;
          if (net_ok) {
#pragma unroll
            for (int i = 1; i < kListLen; i++)
              if (i <= kk) R[i] = (uint32_t)ex_ids[i - 1];
          } else {
            // K + 2 > 16: the list does not fit registers; ids go straight to the output
            int *nn = P.nearest + (long long)gi2 * K;
            for (int i = 0; i < kk; i++) nn[i] = ex_ids[i];
          }
          if (P.stats) atomicAdd(&P.stats[0], 1);
        }
        __syncwarp();
      }
      if (lane == 0) {
        __threadfence_block();
        atomicExch(&misc[M_LOCK], 0);
      }
      __syncwarp();
    }
    __syncwarp();     // the candidate list is dead; its memory becomes the id columns
    if (net_ok) {
#pragma unroll
      for (int i = 1; i < kListLen; i++)
        if (i <= kk) idcol[(i - 1) * kWarp] = (uint16_t)R[i];
    }

    // -------------------------------------------------------------- phase 3: features
    // `fpp` feature planes per pass through the per-warp staging rows (7 planes dx, dy, dspeed,
    // dacc, ddir, type, alive of K columns each, then the time column); each pass leaves by
    // unit-stride row stores
    const int SW = W.sw;
    float *srow = stage + lane * SW;
    int *nn = P.nearest + (long long)gi2 * K;
    // destination row(s) of this lane's agent
    float *dst_obs = (have && P.obs) ? P.obs + (long long)gi2 * F : nullptr;
    float *dst_pol = nullptr;
    if (FUSED && have) {
      const int pol2 = Q.agent_policy[a2], slot2 = Q.agent_slot[a2];
#pragma unroll
      for (int p = 0; p < kMaxPolicies; p++)
        if (p == pol2 && Q.obs_next[p])
          dst_pol = Q.obs_next[p] + ((long long)env * Q.policy_size[p] + slot2) * F;
    }
    const float spa = ssp[a2], acca = sacc[a2], dira = sdir[a2];
    const bool unit_v = (vnorm == 1.0f);
    // destination rows of the warp's 32 agents, once, in the warp's scratch (read back as
    // broadcasts by the copy-out loops) + who is there / alive as ballot masks
    float **rowptr = reinterpret_cast<float **>(s_scr + W.o_rowptr);
    rowptr[2 * lane] = dst_obs;
    rowptr[2 * lane + 1] = dst_pol;
    const unsigned have_mask = __ballot_sync(full, have);
    const unsigned alive_mask = __ballot_sync(full, alive);
    const int n_rows = __popc(have_mask);          // `have` lanes are a prefix of the warp
    __syncwarp();
#pragma unroll 1
    for (int f_lo = 0; f_lo < 7; f_lo += W.fpp) {
      const int f_hi = min(7, f_lo + W.fpp);
      const bool last = (f_hi == 7);
      const int c0 = f_lo * K;
      const int width = (f_hi - f_lo) * K + (last ? 1 : 0);
      if (alive) {
        // one straight loop over the neighbours per feature plane of this pass (:214-250)
#define WDB_PLANE(FI, EXPR)                                                         \
        if (f_lo <= FI && FI < f_hi) {                                              \
          float *col = srow + (FI - f_lo) * K;                                      \
          for (int p = 0; p < K; p++) {                                             \
            float v = 0.0f;                                                         \
            if (p < kk) {                                                           \
              const int b = net_ok ? (int)idcol[p * kWarp] : nn[p];                 \
              if (FI == 0 && net_ok) nn[p] = b;                 /* :202-211 */      \
              v = EXPR;                                                             \
            }                                                                       \
            col[p] = v;                                                             \
          }                                                                         \
        }
        WDB_PLANE(0, div_by_const_f64(pos[b].x - pa.x, diag, inv_diag))
        WDB_PLANE(1, div_by_const_f64(pos[b].y - pa.y, diag, inv_diag))
        WDB_PLANE(2, (unit_v ? ssp[b] - spa : (ssp[b] - spa) / vnorm))
        WDB_PLANE(3, (unit_v ? sacc[b] - acca : (sacc[b] - acca) / vnorm))
        WDB_PLANE(4, div_by_two_pi(sdir[b] - dira, two_pi, inv_two_pi))
        WDB_PLANE(5, (float)stype[b])
        WDB_PLANE(6, (float)salive[b])
#undef WDB_PLANE
        if (last) srow[(7 - f_lo) * K] = static_cast<float>(t_env) / P.episode_length;  // :251-253
      }
      __syncwarp();
      {
        // copy-out: the lanes walk the n_rows x width elements of this pass linearly (row, col
        // advance incrementally), so narrow passes keep all 32 lanes busy
        const int total = n_rows * width;
        const int drow = kWarp / width, dcol = kWarp - drow * width;
        int row = lane / width, col = lane - row * width;
        for (int e = lane; e < total; e += kWarp) {
          const bool r_alive = (alive_mask >> row) & 1u;
          float *o0 = rowptr[2 * row], *o1 = rowptr[2 * row + 1];
          const float v = r_alive ? stage[row * SW + col] : 0.0f;   // dead agents: zero rows
          if (o0) o0[c0 + col] = v;                                  // (:121-139)
          if (o1) o1[c0 + col] = v;
          row += drow;
          col += dcol;
          if (col >= width) { col -= width; row++; }
        }
      }
      __syncwarp();
    }
  } else {
    // full observation (:55-113): one warp per row, lanes over the other agents; rows are
    // dealt over all warps of the cluster
    const int M = N - 1;
    for (int row = warp * C + rank; row < N; row += nw * C) {
      float *orow = P.obs ? P.obs + ((long long)env * N + row) * F : nullptr;
      float *orow2 = nullptr;
      if (FUSED) {
        const int pol = Q.agent_policy[row];
#pragma unroll
        for (int p = 0; p < kMaxPolicies; p++)
          if (p == pol && Q.obs_next[p])
            orow2 = Q.obs_next[p] + ((long long)env * Q.policy_size[p] + Q.agent_slot[row]) * F;
      }
      const bool self_alive = salive[row] != 0;
      for (int idx = lane; idx < M; idx += kWarp) {
        const int b = idx < row ? idx : idx + 1;
        float f0 = 0.f, f1 = 0.f, f2 = 0.f, f3 = 0.f, f4 = 0.f;
        if (self_alive) {
          f0 = div_by_const_f64(pos[b].x - pos[row].x, diag, inv_diag);
          f1 = div_by_const_f64(pos[b].y - pos[row].y, diag, inv_diag);
          f2 = static_cast<float>(ssp[b] - ssp[row]) / vnorm;
          f3 = static_cast<float>(sacc[b] - sacc[row]) / vnorm;
          f4 = div_by_two_pi(sdir[b] - sdir[row], two_pi, inv_two_pi);
        }
        const float f5 = stype[b], f6 = salive[b];
        if (orow) {
          orow[0 * M + idx] = f0; orow[1 * M + idx] = f1; orow[2 * M + idx] = f2;
          orow[3 * M + idx] = f3; orow[4 * M + idx] = f4; orow[5 * M + idx] = f5;
          orow[6 * M + idx] = f6;
        }
        if (orow2) {
          orow2[0 * M + idx] = f0; orow2[1 * M + idx] = f1; orow2[2 * M + idx] = f2;
          orow2[3 * M + idx] = f3; orow2[4 * M + idx] = f4; orow2[5 * M + idx] = f5;
          orow2[6 * M + idx] = f6;
        }
      }
      if (lane == 0) {
        const float tt = self_alive ? static_cast<float>(t_env) / P.episode_length : 0.0f;
        if (orow) orow[7 * M] = tt;
        if (orow2) orow2[7 * M] = tt;
      }
    }
  }

  // ------------------------------------------------------------------ phase 4: rewards / tags
  // (:259-349) thread = agent a2 of the sorted order (any order works: per-agent work)
  float r = 0.0f;
  const bool is_runner = have && (stype[a2] == 0);
  const bool is_alive_now = have && salive[a2] != 0;
  if (is_alive_now) {
    r += scross[a2] ? P.edge_hit_penalty : 0.0f;      // == edge_hit_reward_penalty of this step
    r += P.step_rewards[a2];
  }
  if (is_runner && is_alive_now) {                          // :296-338
    const int tagger = tc_tagging_tagger(P, pos[a2], pos, stag, misc[M_NTAG]);
    if (tagger >= 0) {
      r += P.tag_penalty;
      atomicAdd(&tagcnt[tagger], 1);
      if (P.runner_exits) {
        P.alive[gi2] = 0;
        atomicAdd(&misc[M_EXITS], 1);
      }
      if (P.stats) atomicAdd(&P.stats[1], 1);
    }
    if (t_env == P.episode_length) r += P.end_reward;        // :334-337
  }
  cluster_sync_all();   // #2: every CTA's tag credits and exit counts are final

  // tag credits of my agent (a tagger) and the env's runner count: sums over the cluster
  int credits = 0, exits = 0;
  {
    const uint32_t a_cnt = smem_u32(&tagcnt[a2]), a_ex = smem_u32(&misc[M_EXITS]);
    const bool want = have && stype[a2] == 1;
    for (int rr = 0; rr < C; rr++) {
      if (want) credits += ld_cluster_s32(map_to_rank(a_cnt, (uint32_t)rr));
      exits += ld_cluster_s32(map_to_rank(a_ex, (uint32_t)rr));
    }
  }
  for (int i = 0; i < credits; i++) r += P.tag_reward;      // same float adds as the atomics
  const int nr = g_nrun - exits;
  const int done_now = (t_env == P.episode_length || nr == 0) ? 1 : 0;   // :341-348
  const int d_env = FUSED ? tc_sticky_done(done_now, done_prev) : done_now;
  const bool will_reset = FUSED && d_env && Q.do_reset;
  if (have) P.rewards[gi2] = r;
  if (rank == 0 && tid == 0) {
    P.num_runners[env] = nr;
    if (!will_reset) P.timestep[env] = t_env;
    if (FUSED) tc_book_env(P, Q, env, done_now, done_prev, misc[M_STEPS]);
    else if (done_now) P.done[env] = 1;
  }
  if (FUSED && have) {
    const int pol = Q.agent_policy[a2], slot = Q.agent_slot[a2];
    long long pi = 0;
    float run_prev = 0.0f;
#pragma unroll
    for (int p = 0; p < kMaxPolicies; p++) {
      if (p == pol) {
        pi = (long long)env * Q.policy_size[p] + slot;
        if (Q.reward_running_sum[p]) run_prev = Q.reward_running_sum[p][pi];
      }
    }
    tc_book_agent(Q, pol, pi, r, run_prev, d_env);
  }
  // #3: (a) no CTA may exit while a peer still reads its shared memory; (b) the reset below
  // overwrites rows that other CTAs of the env wrote in this step
  cluster_sync_all();

  // done-masked reset of this env, the words dealt over all threads of the cluster
  if (will_reset)
    tc_reset_env<false>(Q, env, N, F, rank * blockDim.x + tid, C * blockDim.x, warp * C + rank,
                        nw * C, lane);
}

int g_tc_wide_window = 1;   // wdb_set_option("tc_wide_window", 0/1)
int g_tc_wide_bins = 0;     // wdb_set_option("tc_wide_bins", n): 0 = auto
int g_tc_wide_fpp = 0;      // wdb_set_option("tc_wide_fpp", n): feature planes per pass, 0 = auto

inline int align_up(int v, int a) { return (v + a - 1) / a * a; }

template <bool FUSED>
int wide_launch_t(const TcParams &P, const FusedParams &Q, const TcPlan &plan, cudaStream_t st) {
  static size_t configured = 0;
  if (plan.smem > configured) {
    const cudaError_t e = cudaFuncSetAttribute(
        tc_wide_kernel<FUSED>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)plan.smem);
    if (e != cudaSuccess) return (int)e;
    configured = plan.smem;
  }
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3((unsigned)plan.grid, 1, 1);
  cfg.blockDim = dim3((unsigned)plan.block, 1, 1);
  cfg.dynamicSmemBytes = plan.smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[2];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = (unsigned)plan.cluster;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  attr[1].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[1].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = (FUSED && Q.pdl && g_pdl) ? 2 : 1;
  const cudaError_t e = cudaLaunchKernelEx(&cfg, tc_wide_kernel<FUSED>, P, Q, plan.wide);
  if (e != cudaSuccess) return (int)e;
  return finish_launch();
}

}  // namespace

namespace wdb {

int tc_wide_set_option(const char *name, int value, bool *handled) {
  auto is = [&](const char *want) {
    int i = 0;
    for (; want[i] && name[i] == want[i]; i++) {}
    return !want[i] && !name[i];
  };
  *handled = true;
  if (is("tc_wide_window")) { g_tc_wide_window = value ? 1 : 0; return 0; }
  if (is("tc_wide_bins")) {
    if (value < 0 || value > kWideMaxBins || (value & (value - 1))) return (int)cudaErrorInvalidValue;
    g_tc_wide_bins = value;
    return 0;
  }
  if (is("tc_wide_fpp")) {
    if (value < 0 || value > 7) return (int)cudaErrorInvalidValue;
    g_tc_wide_fpp = value;
    return 0;
  }
  *handled = false;
  return 0;
}

// Launch geometry of the cluster kernel; shared-memory carve-up.
int tc_wide_plan(TcParams &P, const FusedParams *Qp, int blocks_per_env, TcPlan &plan) {
  const int N = P.N, K = P.K, C = blocks_per_env;
  if (C < 1 || C > 8) return (int)cudaErrorInvalidValue;        // portable cluster size
  const int S = (N + C - 1) / C;
  const int block = round_up(S, 32);
  if (block > kWideMaxThreads) return (int)cudaErrorInvalidValue;   // needs more CTAs per env
  const int nw = block / 32;
  WideParams W = {};
  W.C = C; W.S = S;
  int nbins = g_tc_wide_bins;
  if (nbins == 0) {
    nbins = 1;
    while (nbins * 16 < N && nbins < kWideMaxBins) nbins <<= 1;   // ~16 agents per bin
  }
  W.nbins = nbins;
  W.npad = round_up(N, 16);
  W.use_window = g_tc_wide_window;
  P.use_history = (g_tc_history && !P.use_full_obs && K + 2 <= kListLen) ? 1 : 0;
  P.force_exact = g_tc_force_exact;
  const int n_chunks = (N + 31) / 32, NB1 = nbins + 1;
  const int list_bytes = (kWideCap + 1) * 32 * 2, id_bytes = (kListLen - 1) * 32 * 2;
  // residency target: 1024 threads per SM; the staging pass width shrinks until that many
  // CTAs fit (the per-CTA copy of the env is what clusters pay for spreading an env out)
  size_t smem = 0;
  int want_ctas = 1024 / block;
  if (want_ctas < 1) want_ctas = 1;
  if (want_ctas > 8) want_ctas = 8;
  static const int kFpp[5] = {7, 4, 3, 2, 1};
  bool fits = false;
  for (; want_ctas >= 1 && !fits; want_ctas--) {
    const size_t budget = (size_t)(227 * 1024) / want_ctas - 1024;
    for (int t = 0; t < 5 && !fits; t++) {
      const int fpp = g_tc_wide_fpp ? g_tc_wide_fpp : kFpp[t];
      int width = 1;                       // widest pass: planes x K (+ the time column)
      for (int f_lo = 0; f_lo < 7; f_lo += fpp) {
        const int f_hi = f_lo + fpp < 7 ? f_lo + fpp : 7;
        const int w = (f_hi - f_lo) * K + (f_hi == 7 ? 1 : 0);
        if (w > width) width = w;
      }
      const int sw = width | 1;
      W.sw = sw; W.fpp = fpp;
      int off = 0;
      auto take = [&](int bytes) { const int o = off; off = align_up(off + bytes, 16); return o; };
      W.o_pos = take(8 * N); W.o_sp = take(4 * N); W.o_acc = take(4 * N); W.o_dir = take(4 * N);
      W.o_alive = take(4 * N); W.o_cross = take(N); W.o_type = take(4 * N);
      W.o_kx = take(4 * W.npad); W.o_ky = take(4 * W.npad); W.o_sid = take(2 * W.npad);
      W.o_tag = take(2 * N);
      const int wc_bytes = 2 * n_chunks * (NB1 + 1);
      W.o_wcount = take(wc_bytes > 4 * N ? wc_bytes : 4 * N);
      W.o_tagcnt = W.o_wcount;            // overlay: the sort table is dead when tags are counted
      W.o_binbase = take(4 * (NB1 + 2)); W.o_leftmax = take(4 * (NB1 + 1));
      W.o_rightmin = take(4 * (NB1 + 1)); W.o_misc = take(4 * M_COUNT);
      W.o_tab = take(4 * (Qp ? Qp->A0 + Qp->A1 : 1));
      W.o_idcol = 0;
      W.o_rowptr = align_up(id_bytes, 16);
      W.stage_warp_bytes = W.o_rowptr + 32 * 2 * 8;          // offset of the staging rows
      int stage_bytes = 4 * 32 * sw;
      if (P.use_full_obs && !Qp) stage_bytes = 16;
      int region = W.stage_warp_bytes + stage_bytes;
      if (region < list_bytes) region = list_bytes;
      if (Qp) {       // the whole scratch holds the lane-strided CDF rows while sampling
        const int amax = Qp->A0 > Qp->A1 ? Qp->A0 : Qp->A1;
        if (region < 128 * amax) region = 128 * amax;
      }
      W.scr_warp_bytes = align_up(region, 16);
      W.o_scr = take(W.scr_warp_bytes * nw);
      W.o_stage = W.o_scr;
      W.o_exact = take(8 * N);
      smem = (size_t)off;
      fits = smem <= budget;
      if (g_tc_wide_fpp) break;
    }
  }
  if (!fits) return (int)cudaErrorInvalidValue;
  if (!P.use_full_obs && !P.obs && !Qp) return (int)cudaErrorInvalidValue;
  plan.kernel = TcPlan::kWide;
  plan.grid = P.n_envs * C;
  plan.block = block;
  plan.cluster = C;
  plan.smem = smem;
  plan.wide = W;
  return 0;
}

int tc_wide_launch(const TcParams &P, const FusedParams *Qp, const TcPlan &plan,
                   cudaStream_t st) {
  if (Qp) return wide_launch_t<true>(P, *Qp, plan, st);
  const FusedParams none = {};
  return wide_launch_t<false>(P, none, plan, st);
}

}  // namespace wdb
