// wdb_tc_small_v2.cu -- second-generation fused / step kernel for SMALL TagContinuous envs
// (EPB whole env replicas per CTA, N <= 128 agents, partial observations, K + 2 <= 16):
// the same mathematics and the same k-nearest selection as tag_continuous_kernel
// (wdb_tag_continuous.cu -- reference tag_continuous_step_pycuda.cu:13-520, core/random.cu:
// 51-85, core/reset.cu:9-75), re-shaped for RESIDENCY.  The first-generation kernel holds the
// whole [EPB, N, F] observation tile (89 KB at config 2) plus the TMA-staged probability
// blocks in shared memory: 113 KB per CTA = 2 CTAs = 20 warps per SM, and its 667 CTAs run as
// 2.5 waves on 132 SMs.  Here
//   * the probabilities are read by their own thread straight from global memory (rows of one
//     policy are contiguous across consecutive threads: every fetched sector is used; L1
//     absorbs the re-touches), the CDF lives in REGISTERS and the reference's binary search
//     (random.cu:33-49) runs on two bit masks (cdf[i] < u, |cdf[i] - u| < 1e-8) -- no
//     probability tile, no CDF rows in shared memory;
//   * the reward / tag phase runs BEFORE the observations are assembled, so the barrier pair
//     around the observation store collapses into the chunk loop;
//   * observations leave through a tile of `chunk_rows` rows that is filled and stored (TMA
//     bulk stores) in passes: each thread assembles its agent's row in the pass the row
//     belongs to.
//   * ALIVE-FIRST working order: runners that were tagged out (about a third of the agents,
//     averaged over a config-2 episode) only need an all-zero observation row.  After the
//     kinematics every env's alive agents take the first slots of the env's thread range
//     (shared-memory counters), the key planes are written compacted, and from the k-nearest
//     selection on thread j of an env works on the agent in slot j: warps that hold only
//     dead agents skip the whole selection, and the candidate scan covers the alive agents
//     only.  Keys carry slot numbers; they are mapped back to agent ids after the
//     verification (the exact path keeps the reference's id order).
// 46-70 KB per CTA -> 3 (EPB = 3) or 4 (EPB = 2) CTAs per SM = 28-30 warps.
// Selected by wdb_set_option("tc_variant", 2); every parity test runs against both variants.
#include "wdb_tc_common.cuh"

namespace {

constexpr int kHistIds = kListLen - 2;   // neighbour ids kept per agent for the threshold

// Register CDF + the reference's binary search on bit masks (A <= W, W = 24 or 32).
template <int W>
__device__ __forceinline__ int sample_row_regs_w(const float *__restrict__ src, int A, float u) {
  float v[W];
#pragma unroll
  for (int i = 0; i < W; i++) v[i] = i < A ? src[i] : 0.0f;
#pragma unroll
  for (int i = 1; i < W; i++) v[i] = v[i] + v[i - 1];     // same left-to-right additions
  uint32_t lt = 0, eq = 0;
#pragma unroll
  for (int i = 0; i < W; i++) {
    if (i < A) {
      if (v[i] < u) lt |= 1u << i;
      if (fabsf(v[i] - u) < 1.0e-8f) eq |= 1u << i;
    }
  }
  int left = 0, right = A - 1;                              // search_index (wdb_common.cuh)
  while (left <= right) {
    const int mid = left + (right - left) / 2;
    if ((eq >> mid) & 1u) return mid;
    if ((lt >> mid) & 1u) left = mid + 1; else right = mid - 1;
  }
  return left > A - 1 ? A - 1 : left;
}
__device__ __forceinline__ int sample_row_regs(const float *__restrict__ src, int A, float u) {
  return A <= 24 ? sample_row_regs_w<24>(src, A, u) : sample_row_regs_w<32>(src, A, u);
}

template <bool FUSED, int MAXT, int MINB>
__global__ void __launch_bounds__(MAXT, MINB)
tc_small_v2_kernel(const __grid_constant__ TcParams P, const __grid_constant__ FusedParams Q,
                   const __grid_constant__ V2Params V) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
#ifdef WDB_PHASE_CLOCKS
  const long long wdb_t0 = clock64();
#endif
  const int N = P.N, epb = P.epb, K = P.K;
  const int EN = epb * N;
  const int nwarps = blockDim.x / kWarp;
  const int Ne = tc_key_stride(N);
  float *skx = reinterpret_cast<float *>(smem_raw);
  float *sky = skx + epb * Ne;
  float2 *spos = reinterpret_cast<float2 *>(sky + epb * Ne);
  float *ssp = reinterpret_cast<float *>(spos + EN);
  float *sacc = ssp + EN;
  float *sdir = sacc + EN;
  float *srew = sdir + EN;
  int *salive = reinterpret_cast<int *>(srew + EN);
  int *stype = salive + EN;       // [N]
  int *stag = stype + N;          // [N]
  int *s_t = stag + N;            // [epb]
  int *s_nrun = s_t + epb;        // [epb]
  int *s_nalive = s_nrun + epb;   // [epb]
  int *s_done = s_nalive + epb;   // [epb]
  int *s_ntag = s_done + epb;     // [4]
  unsigned char *s_scr = smem_raw + tc_small_bytes(epb, N);
  // v2 extras behind the per-warp scratch: tile row -> (env slot << 7 | agent), working slot
  // -> agent id, last step's neighbour ids per agent, then the observation chunk tile
  uint16_t *s_rho = reinterpret_cast<uint16_t *>(s_scr + (size_t)nwarps * P.scr_warp_bytes);
  unsigned char *s_perm = reinterpret_cast<unsigned char *>(s_rho + ((EN + 7) & ~7));
  unsigned char *s_hist = s_perm + ((EN + 15) & ~15);          // [EN][kHistIds]
  int *s_ndead = reinterpret_cast<int *>(s_hist + (((size_t)EN * kHistIds + 15) & ~(size_t)15));
  float *s_tile = reinterpret_cast<float *>(s_ndead + ((epb + 3) & ~3));

  const int tid = threadIdx.x;
  const int lane = tid & 31, warp = tid >> 5;
  const int le = tid / N;
  const int a = tid - le * N;
  const int env0 = blockIdx.x * epb;
  const int env = env0 + le;
  const int envs_here = min(epb, P.n_envs - env0);
  const bool active = (le < epb) && (env < P.n_envs);
  const int gi = env * N + a;
  const int li = le * N + a;
  const float L = P.grid_length;
  const int F = 7 * K + 1;

  // tile rows: per policy p a dense [envs_here, Np] block of rows (one block of all agents in
  // step-only mode) -- the row order of the destination the next forward pass reads
  int row_base[kMaxPolicies];
  {
    int acc = 0;
#pragma unroll
    for (int p = 0; p < kMaxPolicies; p++) {
      row_base[p] = acc;
      if (FUSED && p < Q.n_policies) acc += envs_here * Q.policy_size[p];
    }
  }
  const int total_rows = envs_here * N;

  // ------------------------------------------------------------------ phase 0: all global
  // reads of the prologue back to back, before the first global store
  int g_type = 0;
  if (tid < N) g_type = P.agent_types[tid];
  int my_pol = 0, my_slot = 0;
  if (FUSED && active) { my_pol = Q.agent_policy[a]; my_slot = Q.agent_slot[a]; }
  int pnr[kListLen - 2];
#pragma unroll
  for (int p = 0; p < kListLen - 2; p++)
    pnr[p] = (P.use_history && active && p < K) ? P.nearest[(long long)gi * K + p] : 0;
  float st_x = 0.f, st_y = 0.f, st_sp = 0.f, st_dir = 0.f, st_acc = 0.f, st_skill = 0.f;
  int st_alive = 0;
  if (active) {
    st_x = P.loc_x[gi]; st_y = P.loc_y[gi]; st_sp = P.speed[gi];
    st_dir = P.direction[gi]; st_acc = P.acceleration[gi];
    st_alive = P.alive[gi];
    st_skill = P.skill[a];
  }
  int g_t = 0, g_nrun = 0;
  if (active && a == 0) { g_t = P.timestep[env]; g_nrun = P.num_runners[env]; }
  unsigned long long rng_seed = 0, rng_off = 0;
  float u0 = 0.f, u1 = 0.f;
  if (FUSED && active) {
    if (Q.uniforms) {
      u0 = Q.uniforms[2ll * gi];
      u1 = Q.uniforms[2ll * gi + 1];
    } else {
      rng_seed = reinterpret_cast<const RngHeader *>(Q.rng)->seed;
      rng_off = rng_offsets(Q.rng)[gi];
    }
  }
  float *s_tab = reinterpret_cast<float *>(s_scr);
  const bool tab_ok = FUSED && (size_t)(Q.A0 + Q.A1) * 4 <= (size_t)nwarps * P.scr_warp_bytes;
  float g_tab = 0.f;
  if (tab_ok && tid < Q.A0 + Q.A1)
    g_tab = tid < Q.A0 ? P.acc_actions[tid] : P.turn_actions[tid - Q.A0];
  // probability rows of this agent (fused mode): requested now, consumed after the barrier
  int np_mine = 0;
  const float *g0 = nullptr, *g1 = nullptr;
  if (FUSED && active) {
#pragma unroll
    for (int p = 0; p < kMaxPolicies; p++) {
      if (p == my_pol) {
        np_mine = Q.policy_size[p];
        const long long grow = (long long)env * np_mine + my_slot;
        g0 = Q.probs0[p] + grow * Q.A0;
        g1 = Q.probs1[p] + grow * Q.A1;
      }
    }
  }

  if (tid < N) stype[tid] = g_type;
  if (tab_ok && tid < Q.A0 + Q.A1) s_tab[tid] = g_tab;
  if (tid < epb) { s_nalive[tid] = 0; s_ndead[tid] = 0; }
  for (int i = tid; i < epb * (Ne - N); i += blockDim.x) {   // key padding: never a candidate
    const int e = i / (Ne - N), j = N + (i - e * (Ne - N));
    skx[e * Ne + j] = CUDART_INF_F;
    sky[e * Ne + j] = CUDART_INF_F;
  }
  int rho_own = li;
  if (active) {
    int rho = li;
    if (FUSED) {
#pragma unroll
      for (int p = 0; p < kMaxPolicies; p++)
        if (p == my_pol) rho = row_base[p] + le * Q.policy_size[p] + my_slot;
    }
    s_rho[rho] = (uint16_t)((le << 7) | a);
    rho_own = rho;
    // last step's neighbour ids of this agent, for whichever thread works on it later
#pragma unroll
    for (int p = 0; p < kHistIds; p++)
      s_hist[(size_t)li * kHistIds + p] = (unsigned char)min(max(pnr[p], 0), 127);
  }
  (void)rho_own;
  if (active && a == 0) {
    const int t = g_t + 1;   // :391-393
    P.timestep[env] = t;
    s_t[le] = t;
    s_nrun[le] = g_nrun;
  }
  __syncthreads();     // barrier 0: tables / types / counters staged

  // tagger id list, built by warp 0; read after barrier 1
  if (warp == 0) {
    const int cnt = tc_build_tagger_list(stype, N, stag, lane);
    if (lane == 0) *s_ntag = cnt;
  }

  int act0 = 0, act1 = 0;
  if (FUSED) {
    if (active) {
      if (!Q.uniforms) tc_draw_uniforms(Q, gi, rng_seed, rng_off, u0, u1);
      act0 = sample_row_regs(g0, Q.A0, u0);
      act1 = sample_row_regs(g1, Q.A1, u1);
      tc_push_actions(Q, gi, env, my_pol, np_mine, my_slot, act0, act1);
    }
  } else if (active) {
    const int2 act = *reinterpret_cast<const int2 *>(P.actions + 2ll * gi);
    act0 = act.x; act1 = act.y;
  }

  int alive = 0;
  if (active) {
    alive = st_alive;
    const TcMove mv = tc_move_agent(P, gi, st_x, st_y, st_sp, st_dir, st_acc, st_skill, alive,
                                    tab_ok ? s_tab[act0] : P.acc_actions[act0],
                                    tab_ok ? s_tab[Q.A0 + act1] : P.turn_actions[act1]);
    spos[li] = make_float2(mv.x, mv.y);
    // alive agents take the env's first slots, dead ones the last (any order inside each
    // group: results do not depend on which thread works on which agent)
    const int slot = alive ? atomicAdd(&s_nalive[le], 1) : N - 1 - atomicAdd(&s_ndead[le], 1);
    s_perm[le * N + slot] = (unsigned char)a;
    skx[le * Ne + slot] = alive ? mv.x : CUDART_INF_F;
    sky[le * Ne + slot] = alive ? mv.y : CUDART_INF_F;
    ssp[li] = mv.sp; sacc[li] = mv.acc; sdir[li] = mv.dir;
    salive[li] = alive;
    float r = 0.0f;          // :283-291 reward initialisation (0 + edge + step)
    if (alive) { r += mv.ep; r += P.step_rewards[a]; }
    srew[li] = r;
  }
  __syncthreads();   // barrier 1: state staged; the scratch head (action tables) is dead

  // ------------------------------------------------------------------ k-nearest selection
  const int t_env = active ? s_t[le] : 0;
  const float2 *epos = spos + le * N;
  const int *ealive = salive + le * N;
  // from here on thread (le, j = a) works on the agent in slot j of its env
  const int n_alive = active ? s_nalive[le] : 0;
  const int aw = active ? (int)s_perm[le * N + a] : 0;
  const bool alive_w = active && (a < n_alive);
  const int liw = le * N + aw;
  const int giw = env * N + aw;
  const int nsc = (n_alive + 15) & ~15;            // alive agents fill key slots [0, n_alive)
  const unsigned char *perm = s_perm + le * N;
  uint32_t R[kListLen];
  int kk = 0;
  const bool net_ok = (K + 2 <= kListLen);
  const uint32_t idmask = (1u << P.id_bits) - 1u;
  {
    bool suspect = false;
    if (alive_w) {
      const int nv = n_alive - 1;                 // alive others
      kk = min(nv, K);
      if (net_ok) {
        // fast path: branch-free top-16 of packed (squared distance | id) keys.  Dead
        // agents sit at +inf and sort last; self has key (0 | a).
        const float2 pa = epos[aw];
        const float *kx = skx + le * Ne, *ky = sky + le * Ne;
        uint32_t r0, r1, r2, r3, r4, r5, r6, r7, r8, r9, r10, r11, r12, r13, r14, r15;
        const uint32_t pad_key = 0x7f800000u | idmask;
        bool have = false;          // candidate list already complete (history path)
        float m_out = CUDART_INF_F; // smallest squared distance NOT in the candidate list
        int n_have = min(nv, kListLen - 1);
        int n_cand = nv;            // candidates >= everything the sorted list stands for
        if (P.use_history) {
          // ---- temporal-coherence path.  Threshold tau = the largest current squared
          // distance to last step's neighbours (any tau is safe: the result is accepted
          // only if it provably contains the K nearest, see `hist_ok`).  One pass over
          // the candidates marks everything with s <= tau (typically K + a few) in a
          // 128-bit mask and tracks the minimum of the rest; no sorting network runs over
          // the 100+ candidates.
          float tau = 0.0f;
          int seen = 0;
#pragma unroll
          for (int p = 0; p < kListLen - 2; p++) {
            if (p < K) {
              const int b = min((int)s_hist[(size_t)liw * kHistIds + p], N - 1);
              if (b != aw && ealive[b]) {
                const float2 pb = epos[b];
                tau = fmaxf(tau, sqdist(pa.x, pa.y, pb.x, pb.y));
                seen++;
              }
            }
          }
          // neighbours that left the game shrink the list: widen the disc accordingly
          if (seen < kk) tau *= 1.0f + 0.45f * (float)(kk - seen);
          if (seen == 0) tau = -1.0f;
          WDB_MARK(5)   // tau known
          uint32_t m0 = 0, m1 = 0, m2 = 0, m3 = 0;
          {
            const uint4 *kx4 = reinterpret_cast<const uint4 *>(kx);
            const uint4 *ky4 = reinterpret_cast<const uint4 *>(ky);
            float mo_a = CUDART_INF_F, mo_b = CUDART_INF_F;
#define WDB_SCAN_WORD(W, M)                                                          \
            if (W * 32 < nsc) {                                                      \
              scan_16<0>(M, mo_a, mo_b, kx4 + W * 8, ky4 + W * 8, pa.x, pa.y, tau);  \
              if (W * 32 + 16 < nsc)                                                 \
                scan_16<16>(M, mo_a, mo_b, kx4 + W * 8 + 4, ky4 + W * 8 + 4, pa.x, pa.y, tau); \
            }
            WDB_SCAN_WORD(0, m0) WDB_SCAN_WORD(1, m1) WDB_SCAN_WORD(2, m2) WDB_SCAN_WORD(3, m3)
#undef WDB_SCAN_WORD
            m_out = fminf(mo_a, mo_b);
          }
          WDB_MARK(6)   // scan done
          const int cnt = __popc(m0) + __popc(m1) + __popc(m2) + __popc(m3);
          const bool hist_ok = (cnt >= kk + 1) && (cnt <= kHistCap);   // self + >= kk others
          if (hist_ok) {
            // candidate ids -> this lane's column of the per-warp byte list (rows are kWarp
            // bytes apart), then their keys sorted 16 at a time (slots beyond cnt are stale
            // bytes: clamped and masked to the pad key); one code instance for both halves
            unsigned char *lst = s_scr + (size_t)warp * P.scr_warp_bytes + lane;
            {
              unsigned char *wp = lst;
#define WDB_EXTRACT(M, BASE)                                                         \
              for (uint32_t mm = M; mm; mm &= mm - 1) {                              \
                *wp = (unsigned char)(__ffs(mm) - 1 + BASE);                         \
                wp += kWarp;                                                         \
              }
              WDB_EXTRACT(m0, 0) WDB_EXTRACT(m1, 32) WDB_EXTRACT(m2, 64) WDB_EXTRACT(m3, 96)
#undef WDB_EXTRACT
            }
            WDB_MARK(7)   // ids extracted
#define WDB_HKEY(i)                                                                 \
  uint32_t c##i;                                                                    \
  {                                                                                 \
    const int b = min((int)lst[(hbase + i) * kWarp], N - 1);                        \
    const uint32_t key = (__float_as_uint(sqdist(pa.x, pa.y, kx[b], ky[b])) & ~idmask) \
                         | (uint32_t)b;                                             \
    c##i = (hbase + i < cnt) ? key : pad_key;                                       \
  }
#pragma unroll 1
            for (int hbase = 0; hbase < kHistCap; hbase += kListLen) {
              if (hbase >= cnt) break;
              WDB_REP16(WDB_HKEY)
              WDB_SORT16(c)
              if (hbase == 0) {
                r0 = c0; r1 = c1; r2 = c2; r3 = c3; r4 = c4; r5 = c5; r6 = c6; r7 = c7;
                r8 = c8; r9 = c9; r10 = c10; r11 = c11; r12 = c12; r13 = c13; r14 = c14;
                r15 = c15;
              } else {
                // 17..32 candidates: merge, keeping the 16 smallest (half-cleaner + merger)
                r0 = min(r0, c15); r1 = min(r1, c14); r2 = min(r2, c13); r3 = min(r3, c12);
                r4 = min(r4, c11); r5 = min(r5, c10); r6 = min(r6, c9); r7 = min(r7, c8);
                r8 = min(r8, c7); r9 = min(r9, c6); r10 = min(r10, c5); r11 = min(r11, c4);
                r12 = min(r12, c3); r13 = min(r13, c2); r14 = min(r14, c1); r15 = min(r15, c0);
                WDB_BITONIC_MERGE16(r)
              }
            }
#undef WDB_HKEY
            have = true;
            n_have = min(cnt - 1, kListLen - 1);
            n_cand = cnt - 1;
          } else {
            m_out = CUDART_INF_F;
            if (P.stats) atomicAdd(&P.stats[2], 1);
          }
        }
        if (!have) {
          // rare (first step after a reset, list over/underflow): out-of-line so that the
          // hot path stays small in the instruction cache
          uint32_t out[kListLen];
          network_top16(pa, kx, ky, nsc, idmask, out);
          r0 = out[0]; r1 = out[1]; r2 = out[2]; r3 = out[3]; r4 = out[4]; r5 = out[5];
          r6 = out[6]; r7 = out[7]; r8 = out[8]; r9 = out[9]; r10 = out[10]; r11 = out[11];
          r12 = out[12]; r13 = out[13]; r14 = out[14]; r15 = out[15];
        }   // !have
        R[0] = r0; R[1] = r1; R[2] = r2; R[3] = r3; R[4] = r4; R[5] = r5; R[6] = r6;
        R[7] = r7; R[8] = r8; R[9] = r9; R[10] = r10; R[11] = r11; R[12] = r12;
        R[13] = r13; R[14] = r14; R[15] = r15;
        WDB_MARK(8)   // sorted
        // ---- verification on EXACT float32 squared distances of the K+1 nearest.
        // The network ranked keys whose low id_bits were replaced by the id, so (a) two
        // winners may be mis-ordered when their distances agree in the kept bits -> they
        // are re-sorted exactly below; (b) every candidate the network left out has a
        // squared distance >= floor_out, the key of the last winner with its id bits
        // cleared.  The fast path is valid iff the exact distances are strictly
        // increasing with relative gaps > 2^-19 (so neither the float rounding of
        // dx*dx+dy*dy nor the reference's float(sqrt(double)) can reorder or tie them)
        // and floor_out clears the K-th winner by the same margin.
        const int m = min(n_have, K + 1);
        if ((int)(R[0] & idmask) != a) suspect = true;     // (self sits in key slot j = a)
        float es[kListLen];
        bool misordered = false;
        {
          float prev = 0.0f;
#pragma unroll
          for (int i = 1; i < kListLen; i++) {
            es[i] = CUDART_INF_F;
            if (i <= m) {
              const int c = (int)(R[i] & idmask);              // key slot of the winner
              es[i] = sqdist(pa.x, pa.y, kx[c], ky[c]);
              misordered |= !(es[i] > prev);
              prev = es[i];
            }
          }
        }
        uint32_t last_key = 0;     // R[K + 1] without dynamic register indexing
#pragma unroll
        for (int i = 1; i < kListLen; i++) last_key = (i == K + 1) ? R[i] : last_key;
        const float floor_out = __uint_as_float(last_key & ~idmask);
        if (misordered) {
          // rare: exact odd-even transposition sort of the (<= 15) winners (not unrolled over
          // the passes: code size)
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
          // everything NOT examined above: list entries behind the K+1 winners are
          // >= floor_out (truncated key of winner K+1), candidates outside the list are
          // >= m_out (history path) or >= floor_out (network path, only if nv > 15)
          // (n_cand = others in the candidate list: all alive others on the network path)
          float rest = m_out;
          if (n_cand > K + 1) rest = fminf(rest, floor_out);
          if (rest < CUDART_INF_F && m >= K) {
            float xk = 0.0f;
#pragma unroll
            for (int i = 1; i < kListLen; i++) xk = (i == K) ? es[i] : xk;
            if (!(rest - xk > rest * 1.9073486328125e-06f)) suspect = true;
          }
        }
        // key slots -> agent ids
#pragma unroll
        for (int i = 1; i < kListLen; i++)
          if (i <= kk) R[i] = (uint32_t)perm[min((int)(R[i] & idmask), N - 1)];
      } else {
        suspect = true;
      }
    }
    WDB_MARK(9)   // verified
    if (P.force_exact && alive_w) suspect = true;
    // exact path: the warp resolves its suspect agents one at a time, cooperatively
    unsigned todo = __ballot_sync(0xffffffffu, suspect);
    while (todo) {
      const int Lx = __ffs(todo) - 1;
      todo &= todo - 1;
      const int ax = __shfl_sync(0xffffffffu, aw, Lx);
      const int lex = __shfl_sync(0xffffffffu, le, Lx);
      const int gix = __shfl_sync(0xffffffffu, giw, Lx);
      float *d;
      int *ids;
      if (P.scratch_in_smem) {
        d = reinterpret_cast<float *>(s_scr + (size_t)warp * P.scr_warp_bytes);
        ids = reinterpret_cast<int *>(d + N);
      } else {
        d = P.g_nd + (long long)gix * (N - 1);
        ids = P.g_nid + (long long)gix * (N - 1);
      }
      const int kx = exact_select_warp(spos + lex * N, salive + lex * N, N, ax, K, d, ids, lane);
      if (lane == Lx) {
        kk = kx;
        if (net_ok) {
#pragma unroll
          for (int i = 1; i < kListLen; i++)
            if (i <= kk) R[i] = (uint32_t)ids[i - 1];
        }
        if (P.stats) atomicAdd(&P.stats[0], 1);
      }
      __syncwarp();
    }

    // sorted ids -> this lane's uint16 column of the per-warp scratch (free again: the exact
    // path is done with it), so that the feature loop below is a short runtime loop
    uint16_t *idcol = reinterpret_cast<uint16_t *>(s_scr + (size_t)warp * P.scr_warp_bytes) + lane;
    if (net_ok) {
#pragma unroll
      for (int i = 1; i < kListLen; i++)
        if (i <= kk) idcol[(i - 1) * kWarp] = (uint16_t)(R[i] & idmask);
    }

    if (alive_w && net_ok) {
      int *nn = P.nearest + (long long)giw * K;                   // :202-211
#pragma unroll
      for (int i = 1; i < kListLen; i++)
        if (i <= kk) nn[i - 1] = (int)(R[i] & idmask);
    }
  }

  // policy / slot / tile row of the agent this thread works on
  int pol_w = 0, slot_w = 0, np_w = 0, rho_w = liw;
  if (FUSED && active) {
    pol_w = Q.agent_policy[aw];
    slot_w = Q.agent_slot[aw];
#pragma unroll
    for (int p = 0; p < kMaxPolicies; p++)
      if (p == pol_w) { np_w = Q.policy_size[p]; rho_w = row_base[p] + le * np_w + slot_w; }
  }
  // bookkeeping words needed after the reward phase
  int done_prev = 0, steps_prev = 0;
  float run_prev = 0.0f;
  const long long pi_slot = (long long)env * np_w + slot_w;
  if (FUSED && active) {
    done_prev = P.done[env];
    if (a == 0 && Q.step_running_sum) steps_prev = Q.step_running_sum[env];
#pragma unroll
    for (int p = 0; p < kMaxPolicies; p++)
      if (p == pol_w && Q.reward_running_sum[p]) run_prev = Q.reward_running_sum[p][pi_slot];
  }

  // ------------------------------------------------------------------ rewards / tags (:259-349)
  float r = active ? srew[liw] : 0.0f;
  const bool is_runner = active && (stype[aw] == 0);
  if (is_runner && alive_w) {                                // :296-338
    const int tagger = tc_tagging_tagger(P, epos[aw], epos, stag, *s_ntag);
    if (tagger >= 0) {
      r += P.tag_penalty;
      atomicAdd(&srew[le * N + tagger], P.tag_reward);
      if (P.runner_exits) {
        P.alive[giw] = 0;
        atomicSub(&s_nrun[le], 1);
      }
      if (P.stats) atomicAdd(&P.stats[1], 1);
    }
    if (t_env == P.episode_length) r += P.end_reward;        // :334-337
  }
  __syncthreads();   // barrier 2: tag credits / runner counts final
  int done_now = 0;
  if (active) {
    r = (stype[aw] == 1) ? srew[liw] : r;
    P.rewards[giw] = r;
    const int nr = s_nrun[le];
    done_now = (t_env == P.episode_length || nr == 0) ? 1 : 0;   // :341-348
    if (a == 0) {
      P.num_runners[env] = nr;
      if (FUSED) s_done[le] = tc_book_env(P, Q, env, done_now, done_prev, steps_prev);
      else if (done_now) P.done[env] = 1;
    }
    if (FUSED)
      tc_book_agent(Q, pol_w, pi_slot, r, run_prev, tc_sticky_done(done_now, done_prev));
  }

  // ------------------------------------------------------------------ observations (:29-256)
  // the tile holds `chunk_rows` rows at a time; every thread assembles the row of the agent it
  // works on in the pass that row belongs to (dead agents: an all-zero row, :121-139)
  {
    const double diag = sqrt(2.0) * L;                // :94
    const double inv_diag = 1.0 / diag;
    const float vnorm = P.max_speed + kEpsilon;       // :101
    const float two_pi = kTwoPi, inv_two_pi = 1.0f / kTwoPi;
    const bool unit_v = (vnorm == 1.0f);
    const uint16_t *idcol =
        reinterpret_cast<const uint16_t *>(s_scr + (size_t)warp * P.scr_warp_bytes) + lane;
    const int R_chunk = V.chunk_rows;
    bool tma_pending = false;
    for (int c0 = 0; c0 < total_rows; c0 += R_chunk) {
      const int rows_c = min(R_chunk, total_rows - c0);
      if (c0 > 0) {
        // the TMA engine must have READ the previous chunk before the tile is rewritten
        if (tid == 0 && tma_pending) asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
        __syncthreads();
      }
      if (active && rho_w >= c0 && rho_w < c0 + rows_c) {
        float *orow = s_tile + (rho_w - c0) * F;
        if (!alive_w) {
          for (int f = 0; f < F; f++) orow[f] = 0.0f;
        } else {
          for (int p = kk; p < K; p++) {
#pragma unroll
            for (int f = 0; f < 7; f++) orow[f * K + p] = 0.0f;
          }
          const float2 pa = epos[aw];
          const float spa = ssp[liw], acca = sacc[liw], dira = sdir[liw];
#define WDB_FEATURES(UNIT, UNROLL)                                                  \
          _Pragma(UNROLL)                                                           \
          for (int p = 0; p < kk; p++) {                                            \
            const int b = (int)idcol[p * kWarp];                                    \
            const int lb = le * N + b;                          /* :214-250 */      \
            const float2 pb = epos[b];                                              \
            orow[0 * K + p] = div_by_const_f64(pb.x - pa.x, diag, inv_diag);        \
            orow[1 * K + p] = div_by_const_f64(pb.y - pa.y, diag, inv_diag);        \
            const float dsp = ssp[lb] - spa, dac = sacc[lb] - acca;                 \
            orow[2 * K + p] = UNIT ? dsp : dsp / vnorm;                             \
            orow[3 * K + p] = UNIT ? dac : dac / vnorm;                             \
            orow[4 * K + p] = div_by_two_pi(sdir[lb] - dira, two_pi, inv_two_pi);   \
            orow[5 * K + p] = stype[b];                                             \
            orow[6 * K + p] = ealive[b];                                            \
          }
          if (unit_v) { WDB_FEATURES(true, "unroll 2") } else { WDB_FEATURES(false, "unroll 1") }
#undef WDB_FEATURES
          orow[7 * K] = static_cast<float>(t_env) / P.episode_length;   // :251-253
        }
      }
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
      __syncthreads();   // chunk complete
      // copy-out: every piece (chunk x policy block) with 16-byte aligned addresses and size
      // leaves by TMA, issued by one thread; the others are copied by all threads
      if (!FUSED) {
        float *dst = P.obs + ((long long)env0 * N + c0) * F;
        const uint32_t bytes = 4u * rows_c * F;
        if (tma_ok(dst, smem_u32(s_tile), bytes)) {
          if (tid == 0) {
            tma_store_1d(dst, smem_u32(s_tile), bytes);
            asm volatile("cp.async.bulk.commit_group;" ::: "memory");
          }
          tma_pending = true;
        } else {
          for (int i = tid; i < rows_c * F; i += blockDim.x) dst[i] = s_tile[i];
        }
      } else {
        bool issued = false;
#pragma unroll
        for (int p = 0; p < kMaxPolicies; p++) {
          if (p < Q.n_policies && Q.obs_next[p]) {
            const int np = Q.policy_size[p];
            const int lo = max(c0, row_base[p]), hi = min(c0 + rows_c, row_base[p] + envs_here * np);
            if (lo < hi) {
              const float *src = s_tile + (lo - c0) * F;
              float *dst = Q.obs_next[p] + ((long long)env0 * np + (lo - row_base[p])) * F;
              const uint32_t bytes = 4u * (hi - lo) * F;
              if (tma_ok(dst, smem_u32(src), bytes)) {
                if (tid == 0) tma_store_1d(dst, smem_u32(src), bytes);
                issued = true;
              } else {
                for (int i = tid; i < (hi - lo) * F; i += blockDim.x) dst[i] = src[i];
              }
            }
          }
        }
        if (issued) {
          if (tid == 0) asm volatile("cp.async.bulk.commit_group;" ::: "memory");
          tma_pending = true;
        }
        if (P.obs) {
          // optional [E, N, F] `observations` array: one warp per row
          for (int rr = warp; rr < rows_c; rr += nwarps) {
            const int code = s_rho[c0 + rr];
            const float *src = s_tile + rr * F;
            float *dst = P.obs + ((long long)(env0 + (code >> 7)) * N + (code & 127)) * F;
            for (int f = lane; f < F; f += kWarp) dst[f] = src[f];
          }
        }
      }
    }
    // the TMA stores must have completed before the reset below overwrites the same global
    // rows for finished envs (and have read the tile before the CTA exits)
    if (tid == 0 && tma_pending) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
  }

  if (FUSED && Q.do_reset) {
    // done-masked reset of this CTA's envs (done / timestep already cleared above)
    __syncthreads();   // all global writes of this step by this CTA are issued
    for (int e = 0; e < envs_here; e++)
      if (s_done[e]) tc_reset_env<false>(Q, env0 + e, N, F, tid, blockDim.x, warp, nwarps, lane);
  }
}

int g_tc_v2_threads = 320;   // wdb_set_option("tc_v2_threads", 320 | 224 | 128)

template <bool FUSED, int MAXT, int MINB>
int v2_launch_t(const TcParams &P, const FusedParams &Q, const TcPlan &plan, cudaStream_t st) {
  static size_t configured = 0;
  if (plan.smem > configured) {
    cudaError_t e = cudaFuncSetAttribute(tc_small_v2_kernel<FUSED, MAXT, MINB>,
                                         cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         (int)plan.smem);
    if (e != cudaSuccess) return (int)e;
    cudaFuncSetAttribute(tc_small_v2_kernel<FUSED, MAXT, MINB>,
                         cudaFuncAttributePreferredSharedMemoryCarveout, 100);
    configured = plan.smem;
  }
  tc_small_v2_kernel<FUSED, MAXT, MINB><<<plan.grid, plan.block, plan.smem, st>>>(P, Q, plan.v2);
  return finish_launch();
}

}  // namespace

namespace wdb {

int g_tc_variant = 1;        // wdb_set_option("tc_variant", 1 | 2)

int tc_v2_set_option(const char *name, int value, bool *handled) {
  auto is = [&](const char *want) {
    int i = 0;
    for (; want[i] && name[i] == want[i]; i++) {}
    return !want[i] && !name[i];
  };
  *handled = true;
  if (is("tc_variant")) {
    if (value != 1 && value != 2) return (int)cudaErrorInvalidValue;
    g_tc_variant = value;
    return 0;
  }
  if (is("tc_v2_threads")) {
    if (value != 320 && value != 224 && value != 128) return (int)cudaErrorInvalidValue;
    g_tc_v2_threads = value;
    return 0;
  }
  *handled = false;
  return 0;
}

bool tc_v2_eligible(const TcParams &P, const FusedParams *Q, bool obs_tiles) {
  if (g_tc_variant != 2) return false;
  if (P.use_full_obs || P.K < 1 || P.K + 2 > kListLen || P.N > 128 || P.N < 2) return false;
  if (Q && (Q->A0 > 32 || Q->A1 > 32)) return false;
  return !obs_tiles;
}

int tc_v2_plan(TcParams &P, TcPlan &plan) {
  const int N = P.N, K = P.K, F = 7 * K + 1;
  const int budget_threads = g_tc_v2_threads;
  const int minb = budget_threads == 320 ? 3 : (budget_threads == 224 ? 4 : 7);
  int epb = N >= budget_threads ? 1 : budget_threads / N;
  if (epb > P.n_envs) epb = P.n_envs;
  const int block = round_up(epb * N, 32);
  if (block > budget_threads) return (int)cudaErrorInvalidValue;
  const int nwarps = block / 32, EN = epb * N;
  P.epb = epb;
  P.use_history = g_tc_history ? 1 : 0;
  P.force_exact = g_tc_force_exact;
  size_t warp_bytes = 8ull * N;
  const size_t hist_bytes = (size_t)(kHistCap + 1) * kWarp, id_bytes = (kListLen - 1) * kWarp * 2;
  if (hist_bytes > warp_bytes) warp_bytes = hist_bytes;
  if (id_bytes > warp_bytes) warp_bytes = id_bytes;
  warp_bytes = (warp_bytes + 15) & ~(size_t)15;
  P.scr_warp_bytes = (int)warp_bytes;
  P.scratch_in_smem = 1;
  P.stage_obs = 1;
  int bits = 1;
  while ((1 << bits) < N) bits++;
  P.id_bits = bits;
  // (mirror of the kernel's carve-up: scratch, s_rho, s_perm, s_hist, s_ndead)
  const size_t fixed = tc_small_bytes(epb, N) + warp_bytes * nwarps + (size_t)((EN + 7) & ~7) * 2 +
                       (size_t)((EN + 15) & ~15) +
                       (((size_t)EN * kHistIds + 15) & ~(size_t)15) +
                       (size_t)((epb + 3) & ~3) * 4;
  const size_t budget = (size_t)(227 * 1024) / minb - 1024;     // minb CTAs per SM
  if (fixed + 32ull * F * 4 > budget) return (int)cudaErrorInvalidValue;
  int chunk = (int)((budget - fixed) / (4ull * F)) & ~3;
  const int all_rows = (EN + 3) & ~3;
  if (chunk > all_rows) chunk = all_rows;
  // balance the chunks (same number of chunks, equal sizes)
  const int n_chunks = (EN + chunk - 1) / chunk;
  chunk = (((EN + n_chunks - 1) / n_chunks) + 3) & ~3;
  plan.kernel = TcPlan::kV2;
  plan.v2.chunk_rows = chunk;
  plan.v2.tile_bytes = chunk * F * 4;
  plan.smem = fixed + (size_t)plan.v2.tile_bytes;
  plan.grid = (P.n_envs + epb - 1) / epb;
  plan.block = block;
  plan.minb = minb;
  return 0;
}

int tc_v2_launch(const TcParams &P, const FusedParams *Qp, const TcPlan &plan,
                 cudaStream_t st) {
  const FusedParams none = {};
  if (Qp)
    return plan.minb == 3   ? v2_launch_t<true, 320, 3>(P, *Qp, plan, st)
           : plan.minb == 4 ? v2_launch_t<true, 224, 4>(P, *Qp, plan, st)
                            : v2_launch_t<true, 128, 7>(P, *Qp, plan, st);
  return plan.minb == 3   ? v2_launch_t<false, 320, 3>(P, none, plan, st)
         : plan.minb == 4 ? v2_launch_t<false, 224, 4>(P, none, plan, st)
                          : v2_launch_t<false, 128, 7>(P, none, plan, st);
}

}  // namespace wdb
